"""GPU parity tests (run on an H100 with -m gpu).  Everything goes through the C ABI
(rl4co_b200.native -> libcorollout.so); the checker is the CPU oracle / the golden vectors
recorded from the unmodified reference.

Tolerances (north_star): masks / visited / done / indices bit-exact; rewards and log-probs
1e-5 relative (with a 2e-5 absolute floor for log-probs near 0, since the reference itself is
fp32 and its SDPA/GEMM summation order is unspecified).  Free-running arg-max selections are
compared with near-tie accounting: a GPU choice that differs from the oracle's must be within
TIE_TOL of the oracle's best log-prob *given the same prefix*.
"""

import pytest
import torch

from conftest import env_of
from oracle import am_rollout_oracle as O

pytestmark = pytest.mark.gpu

RTOL, ATOL_LP, TIE_TOL = 1e-5, 2e-5, 1e-4
ENV_FIX = ["env_tsp20", "env_tsp50", "env_cvrp20", "env_cvrp50"]
AM_FIX = ["am_tsp20", "am_cvrp20", "am_tsp50", "am_cvrp50", "am_tsp100", "am_cvrp100"]


@pytest.fixture(scope="module")
def dev():
    from rl4co_b200 import native

    native.lib()  # fail loudly if the extension is missing
    return torch.device("cuda:0")


GEMMS = ["cublas", "tf32x3"]  # strict-fp32 cache GEMM vs the wgmma 3xTF32 kernel


def make_policy(env_name, weights, dev, use_graph_context=True, cache_gemm="cublas", **kw):
    from rl4co_b200.policy import FusedAttentionModelPolicy

    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1, use_graph_context=use_graph_context, **kw)
    pol.decoder.cache_gemm = cache_gemm
    sd = pol.state_dict()
    for k, v in weights.items():
        assert k in sd, f"reference parameter {k} has no counterpart"
        assert sd[k].shape == v.shape, k
    pol.load_state_dict({**sd, **weights})
    return pol.to(dev).eval()


def fused_rollout(pol, env_name, g, dev, decode_type, rows=None, **kw):
    """Run the persistent kernel from golden `h` (encoder output) and instance data."""
    from rl4co_b200 import native
    from rl4co_b200.envs import get_env
    from rl4co_b200.tensordict import TensorDict

    inst = g.inst(dev)
    h = g["h"].to(dev)
    if rows is not None:
        inst = {k: v[:rows] for k, v in inst.items()}
        h = h[:rows]
    env = get_env(env_name, generator_params=dict(num_loc=inst["locs"].shape[1]), check_solution=True)
    td = env.reset(TensorDict(inst, batch_size=[h.shape[0]]))
    pol.encoder = _FixedEncoder(h)
    with torch.inference_mode():
        return pol(td, env, phase="test", decode_type=decode_type, return_sum_log_likelihood=False, **kw), td, env


class _FixedEncoder(torch.nn.Module):
    def __init__(self, h):
        super().__init__()
        self.h = h

    def forward(self, td):
        return self.h, self.h


# ------------------------------------------------------------------------------- env kernels
@pytest.mark.parametrize("name", ENV_FIX)
def test_env_step_kernels_bit_exact(golden, dev, name):
    from rl4co_b200.envs import get_env
    from rl4co_b200.tensordict import TensorDict

    g = golden(name)
    env_name = env_of(name)
    inst = g.inst(dev)
    B = inst["locs"].shape[0]
    env = get_env(env_name, generator_params=dict(num_loc=inst["locs"].shape[1]))
    td = env.reset(TensorDict(inst, batch_size=[B]))
    assert td["done"].shape == (B, 1) and td["done"].dtype == torch.bool
    assert torch.equal(td["action_mask"].cpu(), g["action_mask"][0])
    actions = g["actions"].to(dev)
    for t in range(actions.shape[1]):
        td.set("action", actions[:, t].contiguous())
        td = env.step(td)["next"]
        assert torch.equal(td["action_mask"].cpu(), g["action_mask"][t + 1]), f"mask step {t}"
        assert torch.equal(td["done"].cpu(), g["done"][t])
        assert td["reward"].dtype == torch.bool  # reference quirk: zeros_like(done)
        assert torch.equal(td["current_node"].reshape(-1).cpu(), g["current_node"][t])
        if env_name == "cvrp":
            assert torch.equal(td["visited"].cpu(), g["visited"][t])
            assert torch.equal(td["used_capacity"].cpu(), g["used_capacity"][t])
            assert td["current_node"].shape == (B, 1)
    if env_name == "tsp":
        assert torch.equal(td["first_node"].cpu(), g["first_node"])
        assert torch.equal(td["i"].cpu(), g["i"])
    r = env.get_reward(td, actions)  # includes check_solution_validity
    torch.testing.assert_close(r.cpu(), g["reward"], rtol=RTOL, atol=1e-6)


@pytest.mark.parametrize("name", ENV_FIX)
def test_check_solution_rejects_bad_tours(golden, dev, name):
    from rl4co_b200.envs import get_env
    from rl4co_b200.tensordict import TensorDict

    g = golden(name)
    env_name = env_of(name)
    inst = g.inst(dev)
    env = get_env(env_name, generator_params=dict(num_loc=inst["locs"].shape[1]))
    td = env.reset(TensorDict(inst, batch_size=[inst["locs"].shape[0]]))
    bad = g["actions"].to(dev).clone()
    if env_name == "tsp":
        bad[0, 1] = bad[0, 0]  # node visited twice
    else:
        nz = bad[0].nonzero().reshape(-1)
        bad[0, nz[1]] = bad[0, nz[0]]  # customer visited twice
    with pytest.raises(AssertionError):
        env.check_solution_validity(td, bad)


# ------------------------------------------------------------------------------- decoder step
@pytest.mark.parametrize("name", AM_FIX)
def test_decoder_step_and_select_vs_golden(golden, dev, name):
    """decoder.forward + strategy.step kernels, teacher-forced along the golden greedy path:
    raw logits vs the reference's recorded logits, selection vs recorded actions."""
    from rl4co_b200.decoding import Greedy
    from rl4co_b200.envs import get_env
    from rl4co_b200.tensordict import TensorDict

    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev)
    inst = g.inst(dev)
    B = inst["locs"].shape[0]
    env = get_env(env_name, generator_params=dict(num_loc=inst["locs"].shape[1]))
    td = env.reset(TensorDict(inst, batch_size=[B]))
    td, env, cached = pol.decoder.pre_decoder_hook(td, env, g["h"].to(dev))
    ref_logits, ref_actions, ref_lp = g["greedy_logits"], g["greedy_actions"], g["greedy_logprobs"]
    for t in range(ref_actions.shape[1]):
        logits, mask = pol.decoder(td, cached, 0)
        torch.testing.assert_close(logits.cpu(), ref_logits[t], rtol=1e-4, atol=2e-5)
        assert torch.equal(mask.cpu(), g["greedy_masks"][t])
        strat = Greedy(tanh_clipping=10.0)
        td = strat.step(logits, mask, td)
        lp = strat.logprobs[0].cpu()
        # near-tie aware comparison with the recorded reference selection
        ref_full = O.process_logits(ref_logits[t].clone(), g["greedy_masks"][t])
        chosen = ref_full.gather(1, td["action"].cpu()[:, None]).squeeze(1)
        assert (ref_full.max(1)[0] - chosen < TIE_TOL).all()
        same = td["action"].cpu() == ref_actions[:, t]
        torch.testing.assert_close(lp[same], ref_lp[:, t][same], rtol=RTOL, atol=ATOL_LP)
        td.set("action", ref_actions[:, t].to(dev).contiguous())  # stay on the golden path
        td = env.step(td)["next"]


def test_select_action_modes(dev):
    from rl4co_b200 import native

    torch.manual_seed(0)
    B, N = 257, 101
    logits = torch.randn(B, N) * 3
    mask = torch.rand(B, N) > 0.4
    mask[:, 0] = True
    q = torch.empty(B, N).exponential_(1)
    lp_ref = O.process_logits(logits.clone(), mask)
    lg, mk, qd = logits.to(dev), mask.to(dev), q.to(dev)
    a, lp, full = native.select_action(lg, mk, native.SELECT_GREEDY, store_all_logp=True)
    torch.testing.assert_close(full.cpu(), lp_ref, rtol=RTOL, atol=ATOL_LP)
    assert torch.equal(a.cpu(), full.cpu().argmax(-1))
    a, lp, _ = native.select_action(lg, mk, native.SELECT_SAMPLE_NOISE, noise=qd)
    key = lp_ref.exp() / q
    chosen = key.gather(1, a.cpu()[:, None]).squeeze(1)
    assert (chosen >= key.max(1)[0] * (1 - 1e-5)).all()
    forced = O.select_sampling(lp_ref, mask, q)
    a2, lp2, _ = native.select_action(lg, mk, native.SELECT_EVALUATE, action=forced.to(dev))
    torch.testing.assert_close(lp2.cpu(), lp_ref.gather(1, forced[:, None]).squeeze(1), rtol=RTOL, atol=ATOL_LP)
    a3, _, _ = native.select_action(lg, mk, native.SELECT_SAMPLE_PHILOX, seed=123)
    assert mask.gather(1, a3.cpu()[:, None]).all()


# ------------------------------------------------------------------------------- fused rollout
def _check_against_prefix_oracle(weights, env_name, inst, h, gpu, mode, noise=None, use_graph_context=True,
                                 num_starts=0):
    """Teacher-force the oracle with the GPU's actions; every GPU choice must be the oracle's
    best (or within TIE_TOL of it) under the oracle's own distribution for that prefix, and
    log-probs / reward must agree to tolerance.  Returns the fraction of exactly-equal rows
    against the free-running oracle."""
    acts = gpu["actions"].cpu()
    if num_starts > 1:  # oracle evaluate path works on the expanded batch
        inst = {k: O.batchify(v, num_starts) for k, v in inst.items()}
        h = O.batchify(h, num_starts)
    with torch.inference_mode():
        ref = O.rollout(weights, env_name, inst, h, actions=acts, return_trace=True,
                        use_graph_context=use_graph_context, faithful_copies=False)
    lp_ref = ref["logprobs"]
    lp_gpu = gpu["log_likelihood"].cpu()
    first = 1 if num_starts > 1 else 0
    torch.testing.assert_close(lp_gpu[:, first:], lp_ref[:, first:], rtol=RTOL, atol=ATOL_LP)
    if first:  # forced multistart action carries log-prob 0 (decoding.py:318-323)
        assert (lp_gpu[:, 0] == 0).all()
    torch.testing.assert_close(gpu["reward"].cpu(), ref["reward"], rtol=RTOL, atol=1e-6)
    for t, full in enumerate(ref["trace"]["logprobs"]):
        if t < first:
            continue
        a_t = acts[:, t]
        chosen = full.gather(1, a_t[:, None]).squeeze(1)
        if mode == "greedy":
            assert (full.max(1)[0] - chosen < TIE_TOL).all(), f"step {t}: GPU arg-max is not the oracle's (near-)best"
        elif mode == "sampling":
            key = full.exp() / noise[t]
            kc = key.gather(1, a_t[:, None]).squeeze(1)
            assert (kc >= key.max(1)[0] * (1 - 1e-4)).all(), f"step {t}: GPU sample differs from argmax(p/q)"
    return lp_ref


@pytest.mark.parametrize("gemm", GEMMS)
@pytest.mark.parametrize("name", AM_FIX)
def test_rollout_teacher_forced_vs_golden(golden, dev, name, gemm):
    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev, cache_gemm=gemm)
    out, _, _ = fused_rollout(pol, env_name, g, dev, "evaluate", actions=g["eval_actions"].to(dev))
    torch.testing.assert_close(out["log_likelihood"].cpu(), g["eval_logprobs"], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["reward"].cpu(), g["eval_reward"], rtol=RTOL, atol=1e-6)
    assert torch.equal(out["actions"].cpu(), g["eval_actions"])


def _rows_equal(a, b):
    if a.shape != b.shape:
        return torch.zeros(a.shape[0], dtype=torch.bool)
    return (a == b).all(1)


@pytest.mark.parametrize("gemm", GEMMS)
@pytest.mark.parametrize("name", AM_FIX)
def test_rollout_greedy_vs_golden(golden, dev, name, gemm):
    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev, cache_gemm=gemm)
    out, _, _ = fused_rollout(pol, env_name, g, dev, "greedy")
    _check_against_prefix_oracle(g.weights(), env_name, g.inst(), g["h"], out, "greedy")
    same = _rows_equal(out["actions"].cpu(), g["greedy_actions"])
    # rows that reproduce the recorded trajectory must reproduce its log-probs / reward too
    torch.testing.assert_close(out["log_likelihood"].cpu()[same], g["greedy_logprobs"][same], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["reward"].cpu()[same], g["greedy_reward"][same], rtol=RTOL, atol=1e-6)
    if gemm == "cublas":
        assert same.all(), "golden greedy trajectory not reproduced (near-tie?) -- inspect before relaxing"
    else:  # 1e-6-level cache differences may flip a genuine near-tie (verified above to be one)
        assert same.float().mean() >= 0.75


@pytest.mark.parametrize("gemm", GEMMS)
@pytest.mark.parametrize("name", AM_FIX)
def test_rollout_sampling_recorded_noise_vs_golden(golden, dev, name, gemm):
    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev, cache_gemm=gemm)
    q = g["sampling_noise"]
    T_max = q.shape[2] if env_name == "tsp" else 2 * (q.shape[2] - 1)
    qpad = torch.ones(T_max, q.shape[1], q.shape[2])
    qpad[: q.shape[0]] = q
    out, _, _ = fused_rollout(pol, env_name, g, dev, "sampling", noise=qpad.to(dev))
    _check_against_prefix_oracle(g.weights(), env_name, g.inst(), g["h"], out, "sampling", noise=qpad)
    same = _rows_equal(out["actions"].cpu()[:, : q.shape[0]], g["sampling_actions"])
    torch.testing.assert_close(out["log_likelihood"].cpu()[:, : q.shape[0]][same], g["sampling_logprobs"][same],
                               rtol=RTOL, atol=ATOL_LP)
    assert same.all() if gemm == "cublas" else same.float().mean() >= 0.75


@pytest.mark.parametrize("gemm", GEMMS)
@pytest.mark.parametrize("name", AM_FIX)
@pytest.mark.parametrize("graph_ctx", [True, False])
def test_rollout_multistart_vs_golden(golden, dev, name, graph_ctx, gemm):
    g = golden(name)
    env_name = env_of(name)
    mb = int(g["ms_batch"])
    pol = make_policy(env_name, g.weights(), dev, use_graph_context=graph_ctx, cache_gemm=gemm)
    out, _, _ = fused_rollout(pol, env_name, g, dev, "multistart_greedy", rows=mb)
    key = "ms" if graph_ctx else "pomo"
    assert out["actions"].shape == g[f"{key}_actions"].shape
    inst = {k: v[:mb] for k, v in g.inst().items()}
    S = out["actions"].shape[0] // mb
    _check_against_prefix_oracle(g.weights(), env_name, inst, g["h"][:mb], out, "greedy",
                                 use_graph_context=graph_ctx, num_starts=S)
    same = _rows_equal(out["actions"].cpu(), g[f"{key}_actions"])
    torch.testing.assert_close(out["log_likelihood"].cpu()[same], g[f"{key}_logprobs"][same], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["reward"].cpu()[same], g[f"{key}_reward"][same], rtol=RTOL, atol=1e-6)
    # N = 100: 100 starts x 100 selections per instance -- a genuine near-tie (each verified by the prefix oracle
    # above) flips somewhere even with the strict-fp32 cache
    exact = gemm == "cublas" and g["h"].shape[1] < 100
    assert same.all() if exact else same.float().mean() >= 0.75


@pytest.mark.parametrize("name", AM_FIX)
def test_rollout_multisample_query_batched(golden, dev, name):
    """num_samples > 1 without forced start nodes (decoding.py multisample): S trajectories per
    instance through the query-batched kernel, every column decoded (incl. the TSP placeholder step)."""
    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev)
    S = 6  # not a multiple of the kernel's 4 trajectories per pass: exercises the tail group
    out, _, _ = fused_rollout(pol, env_name, g, dev, "sampling", num_samples=S, seed=9)
    B = g["h"].shape[0]
    assert out["actions"].shape[0] == S * B
    inst = {k: O.batchify(v, S) for k, v in g.inst().items()}
    with torch.inference_mode():
        ref = O.rollout(g.weights(), env_name, inst, O.batchify(g["h"], S), actions=out["actions"].cpu(), faithful_copies=False)
    torch.testing.assert_close(out["log_likelihood"].cpu(), ref["logprobs"], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["reward"].cpu(), ref["reward"], rtol=RTOL, atol=1e-6)
    assert not torch.equal(out["actions"][:B], out["actions"][B:2 * B])  # samples differ across s


@pytest.mark.parametrize("name", ["am_tsp20", "am_cvrp20"])
def test_stepping_path_matches_fused_path(golden, dev, name):
    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev)
    fused, _, _ = fused_rollout(pol, env_name, g, dev, "greedy")
    step, _, _ = fused_rollout(pol, env_name, g, dev, "greedy", fused_rollout=False)
    assert torch.equal(fused["actions"], step["actions"])
    torch.testing.assert_close(fused["log_likelihood"], step["log_likelihood"], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(fused["reward"], step["reward"], rtol=RTOL, atol=1e-6)
    ms_f, _, _ = fused_rollout(pol, env_name, g, dev, "multistart_greedy", rows=3)
    ms_s, _, _ = fused_rollout(pol, env_name, g, dev, "multistart_greedy", rows=3, fused_rollout=False)
    assert torch.equal(ms_f["actions"], ms_s["actions"])


@pytest.mark.parametrize("name", ["am_tsp20", "am_cvrp20"])
@pytest.mark.parametrize("top_k,top_p", [(4, 0.0), (0, 0.8), (6, 0.9)])
def test_stepping_path_top_k_top_p_sampling_vs_oracle(golden, dev, monkeypatch, name, top_k, top_p):
    """decoding.py:109-188 with filters on: the stepping path (kernel per stage + library top-k / sort) under the
    recorded-noise protocol against the free-running oracle; rows may only differ through a genuine near-tie."""
    from rl4co_b200 import decoding

    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev, cache_gemm="cublas")
    q = g["sampling_noise"]
    T_max = q.shape[2] if env_name == "tsp" else 2 * (q.shape[2] - 1)
    qpad = torch.ones(T_max, q.shape[1], q.shape[2])
    qpad[: q.shape[0]] = q
    served = iter(qpad.to(dev))
    monkeypatch.setattr(decoding.Sampling, "_noise", lambda self, logits: next(served).contiguous())
    out, _, _ = fused_rollout(pol, env_name, g, dev, "sampling", top_k=top_k, top_p=top_p)
    with torch.inference_mode():
        ref = O.rollout(g.weights(), env_name, g.inst(), g["h"], decode_type="sampling", top_k=top_k, top_p=top_p,
                        noise=lambda t, shape: qpad[t], faithful_copies=False)
    T = min(out["actions"].shape[1], ref["actions"].shape[1])
    same = _rows_equal(out["actions"].cpu()[:, :T], ref["actions"][:, :T])
    assert same.float().mean() >= 0.75
    torch.testing.assert_close(out["log_likelihood"].cpu()[:, :T][same], ref["logprobs"][:, :T][same], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["reward"].cpu()[same], ref["reward"][same], rtol=RTOL, atol=1e-6)
    if top_k > 0:  # the filter really bites: no step may have chosen outside the k most likely feasible nodes
        assert torch.isfinite(out["log_likelihood"]).all()


@pytest.mark.parametrize("name", ["am_tsp20", "am_cvrp20"])
@pytest.mark.parametrize("beam_width,select_best", [(3, True), (5, False), (None, True)])
def test_stepping_path_beam_search_vs_oracle(golden, dev, name, beam_width, select_best):
    """decoding.py:464-600 on the kernel-per-stage path against the oracle's beam search (itself bit-equal to the live
    reference, tests/test_oracle_vs_reference.py). Beams may only diverge through a near-tie in the top-W cut."""
    g = golden(name)
    env_name = env_of(name)
    pol = make_policy(env_name, g.weights(), dev, cache_gemm="cublas")
    kw = {} if beam_width is None else {"beam_width": beam_width}
    out, _, _ = fused_rollout(pol, env_name, g, dev, "beam_search", select_best=select_best, **kw)
    with torch.inference_mode():
        ref = O.rollout_beam_search(g.weights(), env_name, g.inst(), g["h"], beam_width=beam_width,
                                    select_best=select_best, faithful_copies=False)
    assert out["actions"].shape[0] == ref["actions"].shape[0]
    T = min(out["actions"].shape[1], ref["actions"].shape[1])
    same = _rows_equal(out["actions"].cpu()[:, :T], ref["actions"][:, :T])
    torch.testing.assert_close(out["log_likelihood"].cpu()[:, :T][same], ref["logprobs"][:, :T][same], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["reward"].cpu()[same], ref["reward"][same], rtol=RTOL, atol=1e-6)
    if select_best:
        # several beams of an instance often describe the same tour (routes in another order / direction): the winner
        # among equal-length beams is decided by the last bit of the reward, so compare the winning reward instead
        torch.testing.assert_close(out["reward"].cpu(), ref["reward"], rtol=1e-5, atol=1e-5)
        assert same.float().mean() >= 0.5
    else:
        assert same.float().mean() >= 0.75


# ------------------------------------------------------------------------------- bigger seeded cases
@pytest.mark.parametrize("env_name,n,batch", [("tsp", 100, 96), ("cvrp", 100, 96), ("tsp", 50, 128), ("cvrp", 50, 128),
                                              ("tsp", 7, 33), ("cvrp", 5, 33), ("tsp", 128, 16), ("cvrp", 127, 16),
                                              ("tsp", 33, 40), ("cvrp", 64, 40), ("tsp", 2, 33), ("tsp", 32, 40),
                                              ("tsp", 64, 40), ("cvrp", 31, 40), ("cvrp", 32, 40), ("cvrp", 63, 40)])
@pytest.mark.parametrize("mode", ["greedy", "sampling"])
def test_full_policy_vs_oracle_seeded(dev, env_name, n, batch, mode):
    """Encoder + cache + persistent rollout vs the CPU oracle on seeded instances at the
    BASELINE sizes (N=50/100) and at the slot-boundary sizes of the kernel templates."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(1234 + n)
    env = get_env(env_name, generator_params=dict(num_loc=n), check_solution=True)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2).eval()
    W = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    pol = pol.to(dev)
    td_host = env.generator(batch)
    inst = {k: td_host[k] for k in td_host.keys()}
    N = n + (1 if env_name == "cvrp" else 0)
    T_max = N if env_name == "tsp" else 2 * (N - 1)
    noise = torch.empty(T_max, batch, N).exponential_(1) if mode == "sampling" else None
    kw = {"noise": noise.to(dev)} if noise is not None else {}
    with torch.inference_mode():
        td = env.reset(td_host.to(dev))
        out = pol(td, env, phase="test", decode_type=mode, return_sum_log_likelihood=False, **kw)
        st0 = O.env_reset(env_name, inst)
        h, _ = O.encoder_forward(W, env_name, st0, num_layers=2)
        h_gpu = pol.encoder(td)[0].cpu()
    torch.testing.assert_close(h_gpu, h, rtol=1e-4, atol=1e-4)
    # use the GPU encoder output for the prefix oracle so that decoder parity is isolated
    _check_against_prefix_oracle(W, env_name, inst, h_gpu, out, mode, noise=noise)


@pytest.mark.parametrize("env_name,norm", [("tsp", "batch"), ("cvrp", "instance")])
def test_encoder_tensor_core_path_matches_fp32(dev, env_name, norm):
    """Encoder with its Linear layers on co_gemm_tf32x3 (bias/ReLU/skip/BatchNorm in the GEMM
    epilogue) vs the stock-PyTorch fp32 modules and vs the CPU oracle."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(3)
    env = get_env(env_name, generator_params=dict(num_loc=50))
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=3, normalization=norm).eval()
    for m in pol.modules():  # non-trivial running statistics
        if isinstance(m, torch.nn.BatchNorm1d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    W = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    pol = pol.to(dev)
    td_host = env.generator(300)
    with torch.inference_mode():
        td = env.reset(td_host.to(dev))
        pol.encoder.gemm = "tf32x3"
        h_tc, _ = pol.encoder(td)
        pol.encoder.gemm = "cublas"
        h_fp32, _ = pol.encoder(td)
        st0 = O.env_reset(env_name, {k: td_host[k] for k in td_host.keys()})
        h_ref, _ = O.encoder_forward(W, env_name, st0, num_layers=3, normalization=norm)
    torch.testing.assert_close(h_tc, h_fp32, rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(h_tc.cpu(), h_ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("variant", ["auto", "simt", "wgmma"])
@pytest.mark.parametrize("B,N", [(3, 5), (7, 20), (64, 50), (9, 64), (33, 100), (5, 128), (2, 33), (300, 97), (1, 1),
                                 (17, 65), (4, 72), (11, 81), (6, 104), (2, 121), (269, 127)])
def test_encoder_mha_kernel_vs_sdpa(dev, monkeypatch, variant, B, N):
    """Every attention kernel (all-SIMT, wgmma scores + P.V) against float64 SDPA; B = 300 and 269 make the persistent
    CTAs loop over several instances, and N = 65 .. 127 covers every partial 8-key step of the tensor-core kernel."""
    from rl4co_b200 import native

    if variant == "auto":
        monkeypatch.delenv("CO_MHA_VARIANT", raising=False)
    else:
        monkeypatch.setenv("CO_MHA_VARIANT", variant)
    torch.manual_seed(B * N)
    qkv = torch.randn(B * N, 384, device=dev) * 1.5
    out = native.encoder_mha(qkv, B, N)
    q, k, v = qkv.view(B, N, 3, 8, 16).permute(2, 0, 3, 1, 4).unbind(0)
    ref = torch.nn.functional.scaled_dot_product_attention(q.double(), k.double(), v.double()).transpose(1, 2).reshape(B * N, 128)
    torch.testing.assert_close(out.double(), ref, rtol=1e-5, atol=1e-5 if variant == "simt" else 2e-5)


def test_encoder_mha_rejects_unknown_variant(dev, monkeypatch):
    from rl4co_b200 import native

    monkeypatch.setenv("CO_MHA_VARIANT", "wmma")
    with pytest.raises(native.NativeLibraryError, match="CO_MHA_VARIANT"):
        native.encoder_mha(torch.zeros(4, 384, device=dev), 1, 4)


def test_sampling_philox_is_valid_and_seeded(dev):
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(5)
    env = get_env("cvrp", generator_params=dict(num_loc=50), check_solution=True)
    pol = FusedAttentionModelPolicy(env_name="cvrp", num_encoder_layers=1).to(dev).eval()
    with torch.inference_mode():
        td = env.reset(env.generator(256).to(dev))
        a = pol(td, env, decode_type="sampling", seed=7)   # check_solution=True validates tours
        b = pol(td, env, decode_type="sampling", seed=7)
        c = pol(td, env, decode_type="sampling", seed=8)
    assert torch.equal(a["actions"], b["actions"])
    assert not torch.equal(a["actions"], c["actions"])
    assert (a["log_likelihood"] < 0).all()


def test_sampling_never_selects_masked_nodes_at_scale(dev):
    """2.4e7 in-kernel Exp(1) draws: regression for the u == 1 -> q == 0 -> NaN-key bug (prob 2^-24)."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(0)
    env = get_env("cvrp", generator_params=dict(num_loc=100), check_solution=True)
    pol = FusedAttentionModelPolicy(env_name="cvrp", num_encoder_layers=1).to(dev).eval()
    with torch.inference_mode():
        td = env.reset(env.generator(2048).to(dev))
        for seed in (5, 6):
            pol(td, env, decode_type="sampling", seed=seed)  # check_solution=True raises on an invalid tour


def test_tour_length_properties_full_size(dev):
    """BASELINE-size property checks: reward kernel == in-kernel incremental reward; rotation
    invariance of TSP tours; all tours valid."""
    from rl4co_b200 import native
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(0)
    for env_name, n, B in (("tsp", 100, 8192), ("cvrp", 100, 4096)):
        env = get_env(env_name, generator_params=dict(num_loc=n), check_solution=True)
        pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1).to(dev).eval()
        with torch.inference_mode():
            td = env.reset(env.generator(B).to(dev))
            out = pol(td, env, decode_type="greedy")
            r2 = env.get_reward(td, out["actions"])
        torch.testing.assert_close(out["reward"], r2, rtol=RTOL, atol=1e-5)
        if env_name == "tsp":
            rolled = torch.roll(out["actions"], 17, dims=1).contiguous()
            r3 = native.tour_length(td["locs"], rolled, False)
            torch.testing.assert_close(r3, r2, rtol=RTOL, atol=1e-5)
            ref = O.tsp_reward(td["locs"].cpu(), out["actions"].cpu())
            torch.testing.assert_close(r2.cpu(), ref, rtol=RTOL, atol=1e-5)
        else:
            ref = O.cvrp_reward(td["locs"].cpu(), out["actions"].cpu())
            torch.testing.assert_close(r2.cpu(), ref, rtol=RTOL, atol=1e-5)


def test_reward_stats_kernel(dev):
    from rl4co_b200 import native

    r = torch.randn(100003, device=dev)
    out = torch.zeros(2, dtype=torch.float64, device=dev)
    native.reward_stats(r, out)
    assert abs(out[0].item() - r.double().sum().item()) < 1e-6 * r.numel()
    assert out[1].item() == r.numel()


def test_cpu_tensors_are_rejected_loudly():
    from rl4co_b200 import native
    from rl4co_b200.envs import get_env

    env = get_env("tsp", generator_params=dict(num_loc=10))
    td = env.reset(batch_size=[4])
    td.set("action", torch.zeros(4, dtype=torch.int64))
    with pytest.raises(native.NativeLibraryError):
        env.step(td)


# ------------------------------------------------------------------------------- config C4 at its own scale
def test_pomo_config_c4_vs_reference_fixture(golden, dev):
    """BASELINE config C4 (TSP-100 POMO: 6-layer instance-norm encoder, no graph context, dihedral-8 x 100 starts)
    against `pomo_tsp100.npz`, recorded from the unmodified reference.  (1) decode parity with the oracle-port
    encoder output (pinned to the reference at 1e-5 by tests/test_oracle_golden.py): teacher-forced log-likelihood /
    reward on the reference's 1 600 trajectories <= 1e-5, free-running flips counted and each verified a near-tie;
    (2) the whole GPU policy (hand-written encoder included) through `pomo_step`: POMO's max-over-starts /
    max-over-augs rewards."""
    from conftest import name_seeded_weights
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.reinforce import pomo_step
    from rl4co_b200.tensordict import TensorDict

    g = golden("pomo_tsp100")
    n_aug, seed = int(g["num_augment"]), int(g["weight_seed"])
    pol = FusedAttentionModelPolicy(env_name="tsp", num_encoder_layers=6, normalization="instance",
                                    use_graph_context=False)
    W = name_seeded_weights(pol.state_dict(), seed)
    pol.load_state_dict(W)
    pol = pol.to(dev).eval()
    locs = g["inst::locs"]
    B, N = locs.shape[:2]
    aug = g["aug_locs"]
    ref_actions = g["actions"].long()
    with torch.inference_mode():
        st = O.env_reset("tsp", {"locs": aug})
        h_cpu, _ = O.encoder_forward(W, "tsp", st, num_layers=6, normalization="instance")
    env = get_env("tsp", generator_params=dict(num_loc=N), check_solution=True)
    td = env.reset(TensorDict({"locs": aug.to(dev)}, batch_size=[n_aug * B]))
    # (0) the GPU encoder against the reference rows in the fixture
    with torch.inference_mode():
        h_gpu, _ = pol.encoder(td)
    torch.testing.assert_close(h_gpu[:2].cpu(), g["h_first_rows"], rtol=1e-4, atol=1e-4)
    # (1) decode parity from the oracle's encoder output
    enc = pol.encoder
    pol.encoder = _FixedEncoder(h_cpu.to(dev))
    with torch.inference_mode():
        # teacher forcing works on the expanded batch (one row per trajectory), like the reference's Evaluate
        from rl4co_b200.ops import batchify

        pol.encoder = _FixedEncoder(batchify(h_cpu.to(dev), N))
        ev = pol(batchify(td, N), env, phase="test", actions=ref_actions.to(dev), return_sum_log_likelihood=False)
        pol.encoder = _FixedEncoder(h_cpu.to(dev))
        free = pol(td, env, phase="test", decode_type="multistart_greedy", num_starts=N, return_sum_log_likelihood=False)
    ll = ev["log_likelihood"].cpu()
    torch.testing.assert_close(ll[:, 1:].sum(1), g["logprobs_sum"], rtol=RTOL, atol=5e-5)
    rows = g["logprobs_rows"].shape[0]
    torch.testing.assert_close(ll[:rows, 1:], g["logprobs_rows"][:, 1:], rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(ev["reward"].cpu(), g["reward"], rtol=RTOL, atol=1e-6)
    same = _rows_equal(free["actions"].cpu(), ref_actions)
    flips = int((~same).sum())
    print(f"C4 fixture: {flips} of {same.numel()} free-running trajectories differ from the reference (near-ties)")
    assert same.float().mean() >= 0.9
    torch.testing.assert_close(free["reward"].cpu()[same], g["reward"][same], rtol=RTOL, atol=1e-6)
    _check_against_prefix_oracle(W, "tsp", {"locs": aug}, h_cpu, free, "greedy", use_graph_context=False, num_starts=N)
    # (2) whole GPU policy through the POMO step
    pol.encoder = enc
    td0 = env.reset(TensorDict({"locs": locs.to(dev)}, batch_size=[B]))
    res = pomo_step(pol, env, td0, num_augment=n_aug, num_starts=N, phase="test")
    assert res["reward"].shape == g["reward_b_aug_start"].shape
    # near-tie flips move single trajectories, the best-of-100 / best-of-800 tour lengths barely move
    torch.testing.assert_close(res["max_aug_reward"].cpu(), g["max_aug_reward"], rtol=2e-3, atol=0)
    close = (res["reward"].cpu() - g["reward_b_aug_start"]).abs() <= 1e-5 * g["reward_b_aug_start"].abs()
    assert close.float().mean() >= 0.85


# ------------------------------------------------------------------------------- hygiene (VERDICT r1 #10)
def _chi2(counts, probs):
    n = counts.sum()
    exp = probs * n
    keep = exp > 5
    return (((counts - exp) ** 2 / exp)[keep]).sum().item(), int(keep.sum()) - 1


def test_philox_sampling_distribution_step_kernel(dev):
    """chi-square of the in-kernel Philox draws of `co_select_action` against exp(logp) on a fixed state:
    200 000 independent rows of the same logits (each row is its own Philox stream)."""
    from rl4co_b200 import native

    torch.manual_seed(3)
    N, B = 12, 200_000
    row = torch.randn(N) * 2
    mask_row = torch.ones(N, dtype=torch.bool)
    mask_row[[2, 7]] = False
    logits = row.repeat(B, 1).to(dev)
    mask = mask_row.repeat(B, 1).to(dev)
    p = O.process_logits(row[None].clone(), mask_row[None]).exp()[0].double()
    for seed in (11, 12):
        a, lp, _ = native.select_action(logits, mask, native.SELECT_SAMPLE_PHILOX, seed=seed)
        counts = torch.bincount(a.cpu(), minlength=N).double()
        assert counts[[2, 7]].sum() == 0
        chi2, dof = _chi2(counts, p)
        assert chi2 < 45.0, f"chi2 {chi2:.1f} with {dof} dof (p < 1e-5 at 45 for 9 dof)"  # 9 dof: 99.999 % quantile 37.3


@pytest.mark.parametrize("env_name,temperature", [("tsp", 1.0), ("cvrp", 1.0), ("tsp", 2.0), ("cvrp", 2.0)],
                         ids=["tsp", "cvrp", "tsp-T2", "cvrp-T2"])
def test_philox_sampling_distribution_rollout_kernel(dev, env_name, temperature):
    """The persistent kernel's Gumbel-form sampling (arg-max of z - log q, q = Philox Exp(1), z divided by the
    temperature): B copies of ONE instance, the first free selection of every copy must follow the kernel's own
    reported distribution."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.tensordict import TensorDict

    torch.manual_seed(5)
    n, B = 20, 100_000
    env = get_env(env_name, generator_params=dict(num_loc=n), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1).to(dev).eval()
    for m in pol.decoder.modules():  # sharpen the pointer so that the distribution is far from uniform
        if isinstance(m, torch.nn.Linear):
            m.weight.data *= 3.0
    one = env.generator(1)
    td_host = TensorDict({k: one[k].expand(B, *one[k].shape[1:]).contiguous() for k in one.keys()}, batch_size=[B])
    with torch.inference_mode():
        td = env.reset(td_host.to(dev))
        out = pol(td, env, decode_type="sampling", seed=21, temperature=temperature, return_sum_log_likelihood=False)
    a0, lp0 = out["actions"][:, 0].cpu(), out["log_likelihood"][:, 0].cpu().double()
    N = td["action_mask"].shape[-1]
    counts = torch.bincount(a0, minlength=N).double()
    p = torch.zeros(N, dtype=torch.float64)
    for k in range(N):
        sel = a0 == k
        if sel.any():
            p[k] = lp0[sel].exp().mean()
            assert (lp0[sel] - lp0[sel][0]).abs().max() < 1e-6  # same state -> same reported log-prob
    assert abs(p.sum().item() - 1) < 2e-3  # (nodes never drawn carry < 2e-3 of the mass)
    chi2, dof = _chi2(counts, p / p.sum())
    assert chi2 < 60.0, f"chi2 {chi2:.1f} with {dof} dof"  # <= 20 dof: 99.999 % quantile 56


def test_check_solution_rejects_capacity_overflow(golden, dev):
    """cvrp/env.py:149-177: a tour that visits every customer exactly once but skips a depot return overloads the
    vehicle -- the permutation check passes, the capacity check must fire."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.tensordict import TensorDict

    g = golden("env_cvrp20")
    inst = g.inst(dev)
    B = inst["locs"].shape[0]
    env = get_env("cvrp", generator_params=dict(num_loc=inst["locs"].shape[1]))
    td = env.reset(TensorDict(inst, batch_size=[B]))
    good = g["actions"].to(dev)
    env.check_solution_validity(td, good)  # the recorded tours are valid
    T = good.shape[1]
    bad = good.clone()
    row = bad[0]
    inner = [(t) for t in range(T - 1) if row[t] == 0 and (row[t + 1:] != 0).any() and (row[:t] != 0).any()]
    assert inner, "fixture row 0 has no intermediate depot visit"
    t = inner[0]
    bad[0] = torch.cat([row[:t], row[t + 1:], row.new_zeros(1)])  # drop that depot return (pad with a final depot)
    demand = inst["demand"][0].cpu()
    seg_start = max([u for u in range(t) if row[u] == 0], default=-1) + 1
    nxt = [u for u in range(t + 1, T) if row[u] == 0]
    seg_end = nxt[0] if nxt else T
    load = sum(demand[int(row[u]) - 1] for u in range(seg_start, seg_end) if row[u] != 0)
    assert load > 1.0 + 1e-5, "merged route does not overflow in this fixture row"
    with pytest.raises(AssertionError):
        env.check_solution_validity(td, bad)
