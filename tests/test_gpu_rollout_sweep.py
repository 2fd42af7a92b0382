"""GPU: the persistent whole-episode kernels (`rollout_kernel`, rollout_impl.cuh; the query-batched `rollout_ms_kernel`,
rollout_ms_impl.cuh) against the CPU oracle along the axes random fp32 data at a few fixed sizes does not reach:
temperature and tanh clipping up to the fused path's 2*clip/T < 80 limit, the node-slot boundaries of the sibling envs,
the persistent instance loop, sibling-env multistart, exact ties, and the routing past the fused node limit.

Every check teacher-forces the oracle on the GPU's own actions (`_replay`): per-step log-probs and rewards agree to the
suite's tolerances, a greedy choice is the oracle's best (within TIE_TOL) for the same prefix, a recorded-noise sample is
argmax(p / q). The rollout is fed a fixed encoder output (`encoder_output=`), so a failure points at the rollout kernel.
"""

import pytest
import torch

from oracle import am_rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RTOL, ATOL_LP, TIE_TOL = 1e-5, 2e-5, 1e-4
ENVS = ["tsp", "cvrp", "sdvrp", "op", "pctsp"]
SIBLINGS = ["sdvrp", "op", "pctsp"]


def _num_loc(env_name, N):
    """N is the action-mask width: it counts the depot of the depot envs."""
    return N - 1 if env_name in O.DEPOT_ENVS else N


def _t_max(env_name, N):
    """the fused path's decode-step bound (policy.py)"""
    return {"tsp": N, "cvrp": 2 * (N - 1), "op": N + 1, "pctsp": N + 1}.get(env_name, 3 * (N - 1) + 2)


def _setup(env_name, N, batch, seed, num_layers=1, zero_logits=False):
    """Seeded policy (strict-fp32 cache GEMM), instances, the GPU encoder output and the oracle's view of all three.
    `zero_logits`: the logit third of the node projection (and of the sdvrp dynamic embedding) is zeroed, so that every
    feasible pointer logit is exactly 0."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(seed)
    env = get_env(env_name, generator_params=dict(num_loc=_num_loc(env_name, N)), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=num_layers).eval()
    pol.decoder.cache_gemm = "cublas"
    if zero_logits:
        E = pol.decoder.project_node_embeddings.weight.shape[1]
        with torch.no_grad():
            pol.decoder.project_node_embeddings.weight[2 * E:3 * E] = 0.0
            if env_name == "sdvrp":
                pol.decoder.dynamic_embedding.projection.weight[2 * E:3 * E] = 0.0
    W = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    pol = pol.to(DEV)
    td_host = env.generator(batch)
    inst = {k: td_host[k] for k in td_host.keys()}
    with torch.inference_mode():
        h, _ = pol.encoder(env.reset(td_host.to(DEV)))
    return env, pol, td_host, inst, W, h


def _run(pol, env, td_host, h, **kw):
    with torch.inference_mode():
        return pol(env.reset(td_host.to(DEV)), env, phase="test", return_sum_log_likelihood=False, encoder_output=(h, h),
                   **kw)


def _noise(env_name, N, rows):
    """recorded Exp(1) draws [T_max, rows, N] (the `noise=` protocol: row = s * B + b, one slice per decode step)"""
    return torch.empty(_t_max(env_name, N), rows, N).exponential_(1)


def _record_rollouts(monkeypatch):
    """Route native.rollout through a recorder: one (args, kwargs) entry per co_rollout launch."""
    from rl4co_b200 import native

    calls, real = [], native.rollout

    def recorded(*a, **k):
        calls.append((a, k))
        return real(*a, **k)

    monkeypatch.setattr(native, "rollout", recorded)
    return calls


def _replay(W, env_name, inst, h, acts, num_starts=1, forced_first=False, temperature=1.0, tanh_clipping=10.0):
    """O.rollout's decode loop (constructive/base.py:209-251), teacher-forced on `acts` [B*S, T], keeping the oracle's
    logits, mask and log-prob row of every decoder call. S > 1 rows are start-major over the batchified instances. A
    forced multistart first action is taken by the oracle's *_step without a decoder call and carries log-prob 0
    (decoding.py:309-326) -- O.rollout's evaluate path would score it, and an op start beyond the length budget has
    log-prob -inf there."""
    if num_starts > 1:
        inst, h = O.batchify(inst, num_starts), O.batchify(h, num_starts)
    st = O.env_reset(env_name, inst)
    step_fn = O.ENV_STEP[env_name]
    cache = O.precompute_cache(W, h)
    lps, trace = [], {"mask": [], "logits": [], "logprobs": []}
    t = 0
    if forced_first:
        st = step_fn(st, acts[:, 0])
        lps.append(torch.zeros(acts.shape[0]))
        t = 1
    with torch.inference_mode():
        while not st["done"].all():
            assert t < acts.shape[1], "the GPU trajectories end before the oracle's episode does"
            logits, mask = O.decoder_forward(W, env_name, st, cache, 0, faithful_copies=False)
            lp = O.process_logits(logits.clone(), mask, temperature, tanh_clipping)
            trace["mask"].append(mask)
            trace["logits"].append(logits)
            trace["logprobs"].append(lp)
            lps.append(lp.gather(1, acts[:, t:t + 1]).squeeze(1))
            st = step_fn(st, acts[:, t])
            t += 1
    return {"logprobs": torch.stack(lps, 1), "reward": O.env_reward(env_name, st, acts[:, :t]), "trace": trace,
            "first": 1 if forced_first else 0}


def _check(gpu, ref, mode, noise=None):
    """The suite's prefix-oracle protocol (test_gpu_parity.py) on a `_replay` result."""
    acts, lp_gpu = gpu["actions"].cpu(), gpu["log_likelihood"].cpu()
    first, T = ref["first"], ref["logprobs"].shape[1]
    torch.testing.assert_close(lp_gpu[:, first:T], ref["logprobs"][:, first:], rtol=RTOL, atol=ATOL_LP)
    if first:  # forced multistart action: log-prob 0
        assert (lp_gpu[:, 0] == 0).all()
    # past the oracle's last step every trajectory is done: the kernel pads with the depot at log-prob 0
    assert (acts[:, T:] == 0).all() and (lp_gpu[:, T:] == 0).all()
    torch.testing.assert_close(gpu["reward"].cpu(), ref["reward"], rtol=RTOL, atol=1e-6)
    for t, full in enumerate(ref["trace"]["logprobs"], start=first):
        chosen = full.gather(1, acts[:, t:t + 1]).squeeze(1)
        if mode == "greedy":
            assert (full.max(1)[0] - chosen < TIE_TOL).all(), f"step {t}: GPU arg-max is not the oracle's (near-)best"
        elif mode == "sampling":
            key = full.exp() / noise[t]
            kc = key.gather(1, acts[:, t:t + 1]).squeeze(1)
            assert (kc >= key.max(1)[0] * (1 - 1e-4)).all(), f"step {t}: GPU sample differs from argmax(p/q)"


# ------------------------------------------------------------------------------- A. temperature and tanh clipping
# (10, 0.26): 2*clip/T = 76.9, just inside the fused path's limit, where exp(z - clip/T) nears the bottom of fp32
DECODING = [(10.0, 0.5), (10.0, 2.0), (3.0, 1.0), (25.0, 1.0), (10.0, 0.26)]
A_SIZES = {"tsp": (50, 100), "cvrp": (51, 101), "sdvrp": (41, 90), "op": (51, 101), "pctsp": (51, 101)}


@pytest.mark.parametrize("clip,temp", DECODING)
@pytest.mark.parametrize("env_name,N", [(e, n) for e in ENVS for n in A_SIZES[e]])
def test_decoding_parameters_vs_oracle(env_name, N, clip, temp, monkeypatch):
    """Greedy, recorded-noise sampling and evaluate on the single-trajectory kernel, multistart greedy and multisample
    (the query-batched kernel for tsp / cvrp, the kernel's start loop otherwise), all at the given clip and T."""
    B, S = 12, 4
    env, pol, td_host, inst, W, h = _setup(env_name, N, B, seed=N + int(100 * temp) + int(clip))
    kw = dict(temperature=temp, tanh_clipping=clip)
    rep = dict(temperature=temp, tanh_clipping=clip)
    launches = _record_rollouts(monkeypatch)
    hc = h.cpu()

    out = _run(pol, env, td_host, h, decode_type="greedy", **kw)
    _check(out, _replay(W, env_name, inst, hc, out["actions"].cpu(), **rep), "greedy")

    q = _noise(env_name, N, B)
    smp = _run(pol, env, td_host, h, decode_type="sampling", noise=q.to(DEV), **kw)
    ref = _replay(W, env_name, inst, hc, smp["actions"].cpu(), **rep)
    _check(smp, ref, "sampling", noise=q)
    ev = _run(pol, env, td_host, h, actions=smp["actions"], **kw)
    assert torch.equal(ev["actions"], smp["actions"])
    _check(ev, ref, "evaluate")

    ms = _run(pol, env, td_host, h, decode_type="multistart_greedy", num_starts=S, **kw)
    _check(ms, _replay(W, env_name, inst, hc, ms["actions"].cpu(), num_starts=S, forced_first=True, **rep), "greedy")

    q = _noise(env_name, N, B * S)
    mss = _run(pol, env, td_host, h, decode_type="sampling", num_samples=S, noise=q.to(DEV), **kw)
    _check(mss, _replay(W, env_name, inst, hc, mss["actions"].cpu(), num_starts=S, **rep), "sampling", noise=q)
    assert len(launches) == 5, "a call left the fused path"


@pytest.mark.parametrize("temp,fused", [(0.26, True), (0.25, False)])
@pytest.mark.parametrize("env_name", ENVS)
def test_softmax_limit_routing(env_name, temp, fused, monkeypatch):
    """2*clip/T = 80 exactly (clip 10, T 0.25) takes the stepping path, just inside it the fused kernel; both sides
    match the oracle."""
    N, B = (50 if env_name == "tsp" else 51), 16
    env, pol, td_host, inst, W, h = _setup(env_name, N, B, seed=7)
    launches = _record_rollouts(monkeypatch)
    out = _run(pol, env, td_host, h, decode_type="greedy", temperature=temp, tanh_clipping=10.0)
    assert bool(launches) == fused
    _check(out, _replay(W, env_name, inst, h.cpu(), out["actions"].cpu(), temperature=temp, tanh_clipping=10.0),
           "greedy")


# ------------------------------------------------------------------------------- B. node-slot boundaries
# the smallest instance: one customer; sdvrp needs two, since a one-step episode has no reward in the reference
# (gather_by_index squeezes a one-column action tensor, cvrp/env.py:138-147)
SMALLEST = {"sdvrp": 3, "op": 2, "pctsp": 2}


@pytest.mark.parametrize("mode", ["greedy", "sampling"])
@pytest.mark.parametrize("env_name,N", [(e, n) for e in SIBLINGS for n in (SMALLEST[e], 32, 33, 64, 65, 128)])
def test_sibling_env_slot_edges_vs_oracle(env_name, N, mode):
    """Every slot of a kernel template full (N = 32, 64, 128), one node past it (33, 65), and the smallest instance."""
    B = 24
    env, pol, td_host, inst, W, h = _setup(env_name, N, B, seed=300 + N)
    q = _noise(env_name, N, B) if mode == "sampling" else None
    out = _run(pol, env, td_host, h, decode_type=mode, **({"noise": q.to(DEV)} if q is not None else {}))
    _check(out, _replay(W, env_name, inst, h.cpu(), out["actions"].cpu()), mode, noise=q)


# ------------------------------------------------------------------------------- C. persistent loop
def _instance_rows(B, S, b0, b1):
    """trajectory rows (start-major, s * B + b) of instances b0 .. b1 - 1"""
    return (torch.arange(S)[:, None] * B + torch.arange(b0, b1)[None]).reshape(-1)


def _slice_call(a, k, b0, b1, S):
    """native.rollout arguments of a recorded call restricted to instances b0 .. b1 - 1"""
    B = a[9]
    rows = _instance_rows(B, S, b0, b1).to(DEV)
    a = list(a)
    for i in (2, 3, 6, 7, 8):  # cache, graph context, locs, demand, vehicle capacity: one row per instance
        if a[i] is not None:
            a[i] = a[i][b0:b1].contiguous()
    a[9] = b1 - b0
    k = dict(k)
    for key in ("node_limit", "layer"):  # op / pctsp limits, the EAS-Lay layer: one row per instance
        if k.get(key) is not None:
            k[key] = k[key][b0:b1].contiguous()
    if k.get("forced_actions") is not None:
        k["forced_actions"] = k["forced_actions"][rows].contiguous()
    if k.get("noise") is not None:
        k["noise"] = k["noise"][:, rows].contiguous()
    return a, k


OUT_KEYS = ("actions", "logprobs", "reward", "log_likelihood")


@pytest.mark.parametrize("env_name,S", [("tsp", 1), ("tsp", 6), ("cvrp", 1), ("cvrp", 6), ("sdvrp", 3), ("op", 3),
                                        ("pctsp", 3)])
def test_persistent_loop_batch_composition(env_name, S, monkeypatch):
    """B_inst = 2 * 8 * SMs + 7 makes every CTA of the persistent grid handle at least two instances (it re-initialises
    shared memory, the cvrp demand-rank sort and the sdvrp dynamic terms per instance, and prefetches the next one).
    The same instances in chunks of at most SM-count instances (one per CTA) must give bit-identical actions, per-step
    log-probs, rewards and log-likelihoods. The last 64 instances, which run in a late loop iteration, are checked
    against the oracle."""
    from rl4co_b200 import native

    sms = native.lib().co_device_sm_count()
    B = 2 * 8 * sms + 7
    N = 50 if env_name == "tsp" else 51
    env, pol, td_host, inst, W, h = _setup(env_name, N, B, seed=17 + S)
    calls = _record_rollouts(monkeypatch)
    q = torch.empty(_t_max(env_name, N), B * S, N, device=DEV).exponential_(1)
    greedy = dict(decode_type="multistart_greedy", num_starts=S) if S > 1 else dict(decode_type="greedy")
    multi = dict(num_samples=S) if S > 1 else {}
    g = _run(pol, env, td_host, h, **greedy)
    _run(pol, env, td_host, h, decode_type="sampling", noise=q, **multi)
    _run(pol, env, td_host, h, actions=g["actions"], **multi)
    assert len(calls) == 3
    tail = slice(B - 64, B)
    sub_inst = {k: v[tail] for k, v in inst.items()}
    tail_rows = _instance_rows(B, S, B - 64, B)
    for (a, k), mode in zip(list(calls), ("greedy", "sampling", "evaluate")):
        big = native.rollout(*a, **k)
        chunked = {key: torch.empty_like(big[key]) for key in OUT_KEYS}
        for b0 in range(0, B, sms):
            b1 = min(b0 + sms, B)
            sa, sk = _slice_call(a, k, b0, b1, S)
            res = native.rollout(*sa, **sk)
            rows = _instance_rows(B, S, b0, b1).to(DEV)
            for key in OUT_KEYS:
                chunked[key][rows] = res[key]
        for key in OUT_KEYS:
            assert torch.equal(big[key], chunked[key]), f"{mode}: {key} depends on the batch composition"
        tail_out = {"actions": big["actions"][tail_rows].cpu(), "log_likelihood": big["logprobs"][tail_rows].cpu(),
                    "reward": big["reward"][tail_rows].cpu()}
        forced = mode == "greedy" and S > 1
        ref = _replay(W, env_name, sub_inst, h[tail].cpu(), tail_out["actions"], num_starts=S, forced_first=forced)
        _check(tail_out, ref, mode, noise=q[:, tail_rows.to(DEV)].cpu() if mode == "sampling" else None)


# ------------------------------------------------------------------------------- D. sibling-env multistart
@pytest.mark.parametrize("N", [21, 60])
@pytest.mark.parametrize("env_name", SIBLINGS)
def test_sibling_env_multistart_vs_oracle(env_name, N):
    """The start loop of the single-trajectory kernel (forced starts, the sdvrp demand reload per start) against the
    oracle's *_step replay on the batchified instances. op-20's forced starts may lie beyond the length budget."""
    B = 16
    env, pol, td_host, inst, W, h = _setup(env_name, N, B, seed=40 + N)
    hc = h.cpu()
    for S in (3, 4):
        ms = _run(pol, env, td_host, h, decode_type="multistart_greedy", num_starts=S)
        assert ms["actions"].shape[0] == S * B
        _check(ms, _replay(W, env_name, inst, hc, ms["actions"].cpu(), num_starts=S, forced_first=True), "greedy")
    S = 5
    q = _noise(env_name, N, B * S)
    smp = _run(pol, env, td_host, h, decode_type="sampling", num_samples=S, noise=q.to(DEV))
    _check(smp, _replay(W, env_name, inst, hc, smp["actions"].cpu(), num_starts=S), "sampling", noise=q)


# ------------------------------------------------------------------------------- E. exact ties
def _check_ties(gpu, ref, noise=None):
    """Every feasible logit is exactly 0: greedy must take the lowest feasible index (torch.argmax), a recorded-noise
    sample argmin q over the feasible nodes, each with log-prob -ln(#feasible)."""
    acts, lp_gpu = gpu["actions"].cpu(), gpu["log_likelihood"].cpu()
    first = ref["first"]
    for t, (logits, mask, full) in enumerate(zip(ref["trace"]["logits"], ref["trace"]["mask"], ref["trace"]["logprobs"]),
                                             start=first):
        assert (logits[mask] == 0).all(), "precondition: the oracle's feasible logits are not all 0"
        if noise is None:
            want = mask.int().argmax(1)  # lowest feasible index
            assert torch.equal(full.argmax(1), want)
        else:
            want = torch.where(mask, noise[t], torch.inf).argmin(1)
        assert torch.equal(acts[:, t], want), f"step {t}: tie not resolved like the oracle"
        torch.testing.assert_close(lp_gpu[:, t], -mask.sum(1).double().log().float(), rtol=0, atol=ATOL_LP)


@pytest.mark.parametrize("N", [20, 50, 128])
@pytest.mark.parametrize("env_name", ENVS)
def test_exact_ties_resolve_to_the_lowest_index(env_name, N):
    """Uniform logits on both kernels: within a warp the REDUX.MAX + ballot picks the lowest lane, across the selection
    warps the strict '>' keeps the lower warp."""
    B, S = 16, 4
    env, pol, td_host, inst, W, h = _setup(env_name, N, B, seed=N, zero_logits=True)
    hc = h.cpu()
    out = _run(pol, env, td_host, h, decode_type="greedy")
    ref = _replay(W, env_name, inst, hc, out["actions"].cpu())
    _check_ties(out, ref)
    _check(out, ref, "greedy")
    ms = _run(pol, env, td_host, h, decode_type="multistart_greedy", num_starts=S)
    ref = _replay(W, env_name, inst, hc, ms["actions"].cpu(), num_starts=S, forced_first=True)
    _check_ties(ms, ref)
    _check(ms, ref, "greedy")
    for samples in (1, S):
        q = _noise(env_name, N, B * samples)
        smp = _run(pol, env, td_host, h, decode_type="sampling", noise=q.to(DEV),
                   **({"num_samples": samples} if samples > 1 else {}))
        ref = _replay(W, env_name, inst, hc, smp["actions"].cpu(), num_starts=samples)
        _check_ties(smp, ref, noise=q)
        _check(smp, ref, "sampling", noise=q)


# ------------------------------------------------------------------------------- F. past the fused limit
@pytest.mark.parametrize("env_name", ENVS)
def test_policy_past_the_fused_node_limit(env_name, monkeypatch):
    """N = 129: the stepping kernels and the SDPA branch of the encoder, through the whole policy, against
    O.encoder_forward and the prefix oracle."""
    N, B = 129, 8
    env, pol, td_host, inst, W, h = _setup(env_name, N, B, seed=129, num_layers=2)
    launches = _record_rollouts(monkeypatch)
    with torch.inference_mode():
        out = pol(env.reset(td_host.to(DEV)), env, phase="test", decode_type="greedy", return_sum_log_likelihood=False)
        h_ref, _ = O.encoder_forward(W, env_name, O.env_reset(env_name, inst), num_layers=2)
    assert not launches
    torch.testing.assert_close(h.cpu(), h_ref, rtol=1e-4, atol=1e-4)
    _check(out, _replay(W, env_name, inst, h.cpu(), out["actions"].cpu()), "greedy")


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_policy_beyond_48kb_pointer_shared_memory(env_name):
    """N = 1500: co_pointer_logits opts into more than 48 KB of shared memory (N > 1456)."""
    N = 1500 if env_name == "tsp" else 1501
    env, pol, td_host, inst, W, h = _setup(env_name, N, 2, seed=1500)
    with torch.inference_mode():
        out = pol(env.reset(td_host.to(DEV)), env, phase="test", decode_type="greedy", return_sum_log_likelihood=False)
        h_ref, _ = O.encoder_forward(W, env_name, O.env_reset(env_name, inst), num_layers=1)
    torch.testing.assert_close(h.cpu(), h_ref, rtol=1e-4, atol=1e-4)
    _check(out, _replay(W, env_name, inst, h.cpu(), out["actions"].cpu()), "greedy")
