"""GPU: the search-time kernels -- `co_eas_key_grad`, `co_eas_layer_grad` and the multistart rollout kernel with an
EAS-Lay layer (`co_rollout_args.eas_layer`) or a PolyNet layer (`co_rollout_args.poly`) -- against their float64 oracles
along the axes the tests of each feature (test_gpu_eas.py, test_gpu_eas_layer.py, test_gpu_polynet.py) do not reach:

  A. tanh clipping C and temperature T other than (10, 1).  Both gradient kernels scale the residual by C / (T sqrt(E));
     the rollout computes tanh(u) C / T against the fixed offset C / T.  `eas_search` passes the policy's settings to
     the kernels unchecked, so the gradients are also held to the oracle past the rollout's 2 C / T < 80 limit;
  B. no graph context (POMO's `use_graph_context=False`): the kernels' NULL `graph_ctx` branch;
  C. the persistent instance loop: B = 8 x SMs + 7 instances exceed every grid (at most 8 resident 256-thread CTAs per
     SM), so every CTA handles at least two instances; one call over all of them must be bit-identical to calls over
     chunks of at most SMs instances (one instance per CTA);
  E. exact ties through a layer: a zero logit key makes every feasible pointer logit exactly 0 whatever the layer does.
The node-slot and chunk edges are extra sizes of the per-feature tests.

Tolerances are those of the per-feature tests: per-step log-probs 1e-5 relative / 2e-5 absolute, summed
log-likelihoods 1e-4 absolute, gradients 2e-4 relative Frobenius error (O.gradient_errors) and never all zero, a greedy
step within 2e-5 of the oracle's best.
"""

import dataclasses

import pytest
import torch

from eas_layer_oracle import teacher_forced_logprobs_with_layer
from oracle import am_rollout_oracle as O
from polynet_oracle import rollout_polynet
from test_gpu_eas import _cache, _oracle_grad, _setup
from test_gpu_eas import _grad as _key_grad
from test_gpu_eas import _samples as _key_samples
from test_gpu_eas_layer import _flat, _leaves, _oracle_logprobs, _random_layer
from test_gpu_eas_layer import _grad as _layer_grad
from test_gpu_eas_layer import _rollout as _layer_rollout
from test_gpu_eas_layer import _samples as _layer_samples
from test_gpu_polynet import _check_greedy, _kernel_rollout, _oracle_steps, _recorded_steps, _w64
from test_gpu_polynet import _setup as _poly_setup
from test_gpu_rollout_sweep import OUT_KEYS, _instance_rows, _record_rollouts, _slice_call

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
E = 128
RTOL, ATOL_LP, ATOL_LL, GRAD_TOL = 1e-5, 2e-5, 1e-4, 2e-4
SIZE = {"tsp": 50, "cvrp": 51}  # cvrp: the mask width, depot included

# (10, 0.26): 2 C / T = 76.9, just inside the rollout's fixed-offset softmax limit
DECODING = [(10.0, 0.5), (10.0, 2.0), (3.0, 1.0), (25.0, 1.0), (10.0, 0.26)]
# (10, 0.1): 2 C / T = 200, past that limit; the gradient kernels subtract the row maximum
GRAD_DECODING = DECODING + [(10.0, 0.1)]
NO_GRAPH = (3.0, 1.0)  # B: the setting repeated without a graph context
GRAD_CASES = [(c, t, True) for c, t in GRAD_DECODING] + [(*NO_GRAPH, False)]
ROLL_CASES = [(c, t, True) for c, t in DECODING] + [(*NO_GRAPH, False)]


def _td_host_dict(td_host, sl=slice(None)):
    return {k: td_host[k][sl] for k in td_host.keys()}


# ------------------------------------------------------------------------------- A / B. decoding parameters, graph context
@pytest.mark.parametrize("clip,temp,graph_context", GRAD_CASES)
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_key_gradient_decoding_vs_float64_oracle(env_name, clip, temp, graph_context):
    """co_eas_key_grad at (C, T) on default-setting rows plus an incumbent row, random coefficients."""
    B, S, N = 3, 3, SIZE[env_name]
    dec = dict(tanh_clipping=clip, temperature=temp)
    env, pol, td, td_host = _setup(env_name, N, B, seed=N + int(10 * clip) + int(100 * temp),
                                   use_graph_context=graph_context)
    hidden, cached, cache, L = _cache(pol, td)
    assert (cached.graph_context_or_none is not None) == graph_context
    rows, _ = _key_samples(env_name, pol, td, cached, cache, S, seed=7 * N)
    coef = torch.randn(rows.shape[0], device=DEV)
    dLf, ll = _key_grad(env_name, td, cached, cache, rows, coef, **dec)
    dL = torch.matmul(dLf, pol.decoder.pointer.project_out.weight.t())
    L64, lp = _oracle_grad(pol, env_name, _td_host_dict(td_host), hidden, L, rows, coef, S + 1,
                           use_graph_context=graph_context, **dec)
    torch.testing.assert_close(ll.double().cpu(), lp.sum(1), rtol=RTOL, atol=ATOL_LL)
    rel, zero = O.gradient_errors({"L": dL}, {"L": L64})
    assert not zero and rel["L"] <= GRAD_TOL, rel


@pytest.mark.parametrize("clip,temp,graph_context", GRAD_CASES)
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_layer_gradient_decoding_vs_float64_oracle(env_name, clip, temp, graph_context):
    """co_eas_layer_grad at (C, T) through a non-zero random layer, on rows sampled at the default setting."""
    B, S, N = 3, 3, SIZE[env_name]
    dec = dict(tanh_clipping=clip, temperature=temp)
    env, pol, td, td_host = _setup(env_name, N, B, seed=N + int(10 * clip) + int(100 * temp),
                                   use_graph_context=graph_context)
    hidden, cached, cache, _ = _cache(pol, td)
    assert (cached.graph_context_or_none is not None) == graph_context
    layer = _random_layer(B, seed=3 * N)
    rows = _layer_samples(env_name, td, cached, cache, S, layer, seed=7 * N)
    coef = torch.randn(rows.shape[0], device=DEV)
    dlayer, ll = _layer_grad(env_name, td, cached, cache, rows, coef, layer, **dec)
    leaves = _leaves(layer)
    lp = _oracle_logprobs(pol, env_name, _td_host_dict(td_host), hidden, rows, leaves, S + 1,
                          use_graph_context=graph_context, **dec)
    torch.testing.assert_close(ll.double().cpu(), lp.sum(1).detach(), rtol=RTOL, atol=ATOL_LL)
    (coef.double().cpu() * lp.sum(1)).sum().backward()
    got = {k: v.reshape(leaves[k].shape) for k, v in _flat(dlayer).items()}
    rel, zero = O.gradient_errors(got, leaves)
    assert not zero and max(rel.values()) <= GRAD_TOL, rel


@pytest.mark.parametrize("clip,temp,graph_context", ROLL_CASES)
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_rollout_with_layer_decoding_vs_oracle(env_name, clip, temp, graph_context):
    """The LAYER rollout at (C, T): Philox-sampled tours are valid and carry the oracle's teacher-forced log-probs
    through the layer; evaluate mode on tours sampled without the layer likewise."""
    from rl4co_b200 import native

    B, S, N = 3, 5, SIZE[env_name]
    dec = dict(tanh_clipping=clip, temperature=temp)
    ora = dict(use_graph_context=graph_context, **dec)
    env, pol, td, td_host = _setup(env_name, N, B, seed=N + int(10 * clip) + int(100 * temp),
                                   use_graph_context=graph_context)
    hidden, cached, cache, _ = _cache(pol, td)
    layer = _random_layer(B, seed=N)
    inst = _td_host_dict(td_host)
    leaves = {k: v.detach() for k, v in _leaves(layer).items()}
    vrp = env_name == "cvrp"
    out = _layer_rollout(env_name, td, cached, cache, S, layer, seed=N, **dec)
    assert native.check_tours(out["actions"], N, td["demand"].contiguous() if vrp else None,
                              td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None, B_inst=B) == 0
    with torch.no_grad():
        ref = _oracle_logprobs(pol, env_name, inst, hidden, out["actions"], leaves, S, **ora)
    torch.testing.assert_close(out["logprobs"][:, :ref.shape[1]].double().cpu(), ref, rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["log_likelihood"].double().cpu(), ref.sum(1), rtol=RTOL, atol=ATOL_LL)
    rows = _layer_rollout(env_name, td, cached, cache, S, None, seed=N + 1)["actions"].contiguous()
    ev = _layer_rollout(env_name, td, cached, cache, S, layer, mode=native.SELECT_EVALUATE, forced=rows, **dec)
    assert torch.equal(ev["actions"], rows)
    with torch.no_grad():
        ref = _oracle_logprobs(pol, env_name, inst, hidden, rows, leaves, S, **ora)
    torch.testing.assert_close(ev["logprobs"][:, :ref.shape[1]].double().cpu(), ref, rtol=RTOL, atol=ATOL_LP)


def _poly_policy_checks(env_name, N, clip, temp, graph_context, seed, sampling=True):
    """FusedPolyNetPolicy(temperature=T, tanh_clipping=C), k = 3, S = 9: greedy (the `_check_greedy` protocol) and
    recorded-noise sampling against `rollout_polynet`."""
    k, S, B = 3, 9, 2
    dec = dict(tanh_clipping=clip, temperature=temp)
    ora = dict(use_graph_context=graph_context, **dec)
    env, pol, td, inst = _poly_setup(env_name, N, B, k, seed=seed, use_graph_context=graph_context, **dec)
    with torch.inference_mode():
        out = pol(td, env, phase="test", decode_type="greedy", num_starts=S, return_sum_log_likelihood=False,
                  return_hidden=True)
    acts = out["actions"].cpu()
    h64 = out["hidden"].double().cpu()
    lp64, full64 = _oracle_steps(_w64(pol), env_name, inst, h64, acts, S, **ora)
    _check_greedy(out["log_likelihood"], acts, lp64, full64)
    if not sampling:
        return
    T = N if env_name == "tsp" else 2 * (N - 1)
    q = torch.empty(T, B * S, N).exponential_(1, generator=torch.Generator().manual_seed(seed))
    with torch.inference_mode():
        smp = pol(td, env, phase="train", decode_type="sampling", num_starts=S, noise=q.to(DEV),
                  return_sum_log_likelihood=False, return_hidden=True)
    h64 = smp["hidden"].double().cpu()
    ref = rollout_polynet(_w64(pol), env_name, inst, h64, decode_type="multistart_sampling", num_starts=S,
                          noise=lambda step, shape: q[step].double(), **ora)
    T = ref["actions"].shape[1]
    same = (smp["actions"].cpu()[:, :T] == ref["actions"]).all(1)
    assert float(same.float().mean()) >= 0.95, f"only {float(same.float().mean()):.0%} of the rows sampled alike"
    torch.testing.assert_close(smp["log_likelihood"].cpu()[same, :T].double(), ref["logprobs"][same], rtol=RTOL,
                               atol=ATOL_LP)


@pytest.mark.parametrize("clip,temp,graph_context", ROLL_CASES)
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_polynet_decoding_vs_oracle(env_name, clip, temp, graph_context, monkeypatch):
    """The POLY rollout at (C, T), through the policy; both decodes run the fused kernel."""
    launches = _record_rollouts(monkeypatch)
    _poly_policy_checks(env_name, SIZE[env_name], clip, temp, graph_context, seed=int(10 * clip) + int(100 * temp))
    assert len(launches) == 2, "a decode left the fused path"


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_polynet_past_the_softmax_limit_takes_the_stepping_path(env_name, monkeypatch):
    """2 C / T = 80 exactly (C 10, T 0.25): the policy decodes greedily on the stepping path (which takes no recorded
    noise), matching the oracle too."""
    launches = _record_rollouts(monkeypatch)
    _poly_policy_checks(env_name, SIZE[env_name], 10.0, 0.25, True, seed=25, sampling=False)
    assert not launches


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_null_graph_context_equals_a_zero_graph_context(env_name):
    """Without a graph context all four paths take their NULL `graph_ctx` branch, which must compute exactly what an
    explicit all-zero context computes (x + 0 == x in fp32).  Bit for bit, this sees a stray term in that branch that
    the oracle tolerances cannot: a 1e-3 offset on every query channel of the key gradient stays near 5e-5 relative
    gradient error, under the 2e-4 bound."""
    from rl4co_b200 import native

    B, S, N = 3, 3, SIZE[env_name]
    dec = dict(tanh_clipping=NO_GRAPH[0], temperature=NO_GRAPH[1])
    env, pol, td, _ = _setup(env_name, N, B, seed=90, use_graph_context=False)
    hidden, cached, cache, _ = _cache(pol, td)
    assert cached.graph_context_or_none is None
    zero = dataclasses.replace(cached, graph_context=torch.zeros(B, E, device=DEV))
    rows, _ = _key_samples(env_name, pol, td, cached, cache, S, seed=91)
    coef = torch.randn(rows.shape[0], device=DEV)
    layer = _random_layer(B, seed=92)
    for name, run in (("key gradient", lambda c: _key_grad(env_name, td, c, cache, rows, coef, **dec)),
                      ("layer gradient", lambda c: _layer_grad(env_name, td, c, cache, rows, coef, layer, **dec)),
                      ("layer rollout", lambda c: _layer_rollout(env_name, td, c, cache, S, layer, seed=93, **dec))):
        a, b = run(cached), run(zero)
        for x, y in (zip(a, b) if isinstance(a, tuple) else ((a[k], b[k]) for k in OUT_KEYS)):
            assert torch.equal(x, y), f"{name}: a NULL graph context differs from a zero one"
    k = 3
    env, pol, td, _ = _poly_setup(env_name, N, B, k, seed=94, use_graph_context=False, **dec)
    with torch.inference_mode():
        cached = pol.decoder._precompute_cache(pol.encoder(td)[0])
        assert cached.graph_context_or_none is None
        zero = dataclasses.replace(cached, graph_context=torch.zeros(B, E, device=DEV))
        for mode in (native.SELECT_GREEDY, native.SELECT_SAMPLE_PHILOX):
            a = _kernel_rollout(env_name, pol, td, cached, 2 * k, mode)
            b = _kernel_rollout(env_name, pol, td, zero, 2 * k, mode)
            for key in OUT_KEYS:
                assert torch.equal(a[key], b[key]), f"poly rollout: a NULL graph context differs from a zero one ({key})"


# ------------------------------------------------------------------------------- C. persistent instance loop
TAIL = 16  # instances held to the oracle: the last ones, which run in the loop's last iteration


def _persistent_batch():
    from rl4co_b200 import native

    sms = native.lib().co_device_sm_count()
    return 8 * sms + 7, sms


def _chunks(B, sms):
    return [(b0, min(b0 + sms, B)) for b0 in range(0, B, sms)]


def _sub_cached(cached, b0, b1):
    g = cached.graph_context_or_none
    return type(cached)(node_embeddings=cached.node_embeddings[b0:b1],
                        graph_context=g[b0:b1] if g is not None else cached.graph_context, rollout_cache=None,
                        q_placeholder=cached.q_placeholder, w_capacity=cached.w_capacity)


def _sub_td(env_name, td, b0, b1):
    return {k: td[k][b0:b1] for k in (("demand", "vehicle_capacity") if env_name == "cvrp" else ())}


def _grad_chunked(grad_fn, env_name, td, cached, cache, rows, coef, B, R, sms, layer=None):
    """`grad_fn` over instances b0 .. b1 - 1 of every chunk -> (per-instance gradient [B, ...], loglik [R * B])."""
    extra = {}
    outs_d, ll = [], torch.empty_like(coef)
    for b0, b1 in _chunks(B, sms):
        sel = _instance_rows(B, R, b0, b1).to(DEV)
        if layer is not None:
            extra = dict(layer=layer[b0:b1].contiguous())
        d, l_ = grad_fn(env_name, _sub_td(env_name, td, b0, b1), _sub_cached(cached, b0, b1),
                        cache[b0:b1].contiguous(), rows[sel].contiguous(), coef[sel].contiguous(), **extra)
        outs_d.append(d)
        ll[sel] = l_
    return torch.cat(outs_d), ll


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_key_gradient_persistent_loop_batch_composition(env_name):
    B, sms = _persistent_batch()
    S, N = 3, SIZE[env_name]
    R = S + 1
    env, pol, td, td_host = _setup(env_name, N, B, seed=61)
    hidden, cached, cache, L = _cache(pol, td)
    rows, _ = _key_samples(env_name, pol, td, cached, cache, S, seed=62)
    coef = torch.randn(rows.shape[0], device=DEV)
    dLf, ll = _key_grad(env_name, td, cached, cache, rows, coef)
    dc, lc = _grad_chunked(_key_grad, env_name, td, cached, cache, rows, coef, B, R, sms)
    assert torch.equal(dLf, dc), "dLf depends on the batch composition"
    assert torch.equal(ll, lc), "loglik depends on the batch composition"
    tail, sel = slice(B - TAIL, B), _instance_rows(B, R, B - TAIL, B).to(DEV)
    L64, lp = _oracle_grad(pol, env_name, _td_host_dict(td_host, tail), hidden[tail], L[tail], rows[sel], coef[sel], R)
    torch.testing.assert_close(ll[sel].double().cpu(), lp.sum(1), rtol=RTOL, atol=ATOL_LL)
    dL = torch.matmul(dLf[tail], pol.decoder.pointer.project_out.weight.t())
    rel, zero = O.gradient_errors({"L": dL}, {"L": L64})
    assert not zero and rel["L"] <= GRAD_TOL, rel


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_layer_gradient_persistent_loop_batch_composition(env_name):
    B, sms = _persistent_batch()
    S, N = 3, SIZE[env_name]
    R = S + 1
    env, pol, td, td_host = _setup(env_name, N, B, seed=63)
    hidden, cached, cache, _ = _cache(pol, td)
    layer = _random_layer(B, seed=64)
    rows = _layer_samples(env_name, td, cached, cache, S, layer, seed=65)
    coef = torch.randn(rows.shape[0], device=DEV)
    dlayer, ll = _layer_grad(env_name, td, cached, cache, rows, coef, layer)
    dc, lc = _grad_chunked(_layer_grad, env_name, td, cached, cache, rows, coef, B, R, sms, layer=layer)
    assert torch.equal(dlayer, dc), "dlayer depends on the batch composition"
    assert torch.equal(ll, lc), "loglik depends on the batch composition"
    tail, sel = slice(B - TAIL, B), _instance_rows(B, R, B - TAIL, B).to(DEV)
    leaves = _leaves(layer[tail])
    lp = _oracle_logprobs(pol, env_name, _td_host_dict(td_host, tail), hidden[tail], rows[sel], leaves, R)
    torch.testing.assert_close(ll[sel].double().cpu(), lp.sum(1).detach(), rtol=RTOL, atol=ATOL_LL)
    (coef[sel].double().cpu() * lp.sum(1)).sum().backward()
    got = {k: v.reshape(leaves[k].shape) for k, v in _flat(dlayer[tail]).items()}
    rel, zero = O.gradient_errors(got, leaves)
    assert not zero and max(rel.values()) <= GRAD_TOL, rel


def _rollout_modes(call, B, S, N, T_max):
    """Greedy, recorded-noise sampling and evaluate (on the greedy tours) variants of one recorded `native.rollout`
    greedy call -> [(mode, args, kwargs)]."""
    from rl4co_b200 import native

    a, k = call
    greedy = native.rollout(*a, **k)
    smp = list(a)
    smp[1] = native.SELECT_SAMPLE_NOISE
    ev = list(a)
    ev[1] = native.SELECT_EVALUATE
    q = torch.empty(T_max, B * S, N, device=DEV).exponential_(1, generator=torch.Generator(DEV).manual_seed(N))
    return [("greedy", a, k), ("sampling", smp, dict(k, noise=q)),
            ("evaluate", ev, dict(k, forced_actions=greedy["actions"].contiguous()))]


def _check_batch_composition(a, k, mode, B, S, sms):
    """One `native.rollout(*a, **k)` call over all B instances against calls over chunks of at most `sms` instances:
    bit-identical outputs.  Returns the whole call's outputs."""
    from rl4co_b200 import native

    big = native.rollout(*a, **k)
    chunked = {key: torch.empty_like(big[key]) for key in OUT_KEYS}
    for b0, b1 in _chunks(B, sms):
        sa, sk = _slice_call(a, k, b0, b1, S)
        res = native.rollout(*sa, **sk)
        rows = _instance_rows(B, S, b0, b1).to(DEV)
        for key in OUT_KEYS:
            chunked[key][rows] = res[key]
    for key in OUT_KEYS:
        assert torch.equal(big[key], chunked[key]), f"{mode}: {key} depends on the batch composition"
    return big


def _check_tail(big, mode, B, S, replay):
    """The last TAIL instances of a persistent-loop call against the oracle: `replay(acts)` -> (float64 log-probs,
    full log-prob rows) of their S forced-start rows, start-major."""
    rows = _instance_rows(B, S, B - TAIL, B).to(DEV)
    acts = big["actions"][rows].cpu()
    lp64, full64 = replay(acts)
    T = lp64.shape[1]
    if mode == "greedy":
        _check_greedy(big["logprobs"][rows], acts, lp64, full64)
    else:
        torch.testing.assert_close(big["logprobs"][rows][:, :T].double().cpu(), lp64, rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(big["log_likelihood"][rows].double().cpu(), lp64.sum(1), rtol=RTOL, atol=ATOL_LL)


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_rollout_with_layer_persistent_loop_batch_composition(env_name, monkeypatch):
    from rl4co_b200 import native

    B, sms = _persistent_batch()
    S, N = 3, SIZE[env_name]
    T_max = N if env_name == "tsp" else 2 * (N - 1)
    env, pol, td, td_host = _setup(env_name, N, B, seed=66)
    hidden, cached, cache, _ = _cache(pol, td)
    layer = _random_layer(B, seed=67)
    calls = _record_rollouts(monkeypatch)
    _layer_rollout(env_name, td, cached, cache, S, layer, mode=native.SELECT_GREEDY)
    tail = slice(B - TAIL, B)
    W64 = O.float64_weights(pol.state_dict(), ())
    inst, h64 = _td_host_dict(td_host, tail), hidden[tail].double().cpu()
    leaves = {k: v.detach() for k, v in _leaves(layer[tail]).items()}

    def replay(acts):
        return _recorded_steps(teacher_forced_logprobs_with_layer, W64, env_name, inst, h64, acts, leaves,
                               num_starts=S, forced_first=True)

    for mode, a, k in _rollout_modes(calls[0], B, S, N, T_max):
        big = _check_batch_composition(a, k, mode, B, S, sms)
        with torch.no_grad():
            _check_tail(big, mode, B, S, replay)


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_polynet_rollout_persistent_loop_batch_composition(env_name, monkeypatch):
    from rl4co_b200 import native

    B, sms = _persistent_batch()
    k, S, N = 4, 6, SIZE[env_name]
    T_max = N if env_name == "tsp" else 2 * (N - 1)
    env, pol, td, inst = _poly_setup(env_name, N, B, k, seed=68)
    with torch.inference_mode():
        hidden = pol.encoder(td)[0]
        cached = pol.decoder._precompute_cache(hidden)
        calls = _record_rollouts(monkeypatch)
        _kernel_rollout(env_name, pol, td, cached, S, native.SELECT_GREEDY)
        modes = _rollout_modes(calls[0], B, S, N, T_max)
        bigs = [(mode, _check_batch_composition(a, kw, mode, B, S, sms)) for mode, a, kw in modes]
    tail = slice(B - TAIL, B)
    W64, h64 = _w64(pol), hidden[tail].double().cpu()
    inst = {key: v[tail] for key, v in inst.items()}
    for mode, big in bigs:
        _check_tail(big, mode, B, S, lambda acts: _oracle_steps(W64, env_name, inst, h64, acts, S))


# ------------------------------------------------------------------------------- E. exact ties through a layer
def _check_ties(lp_gpu, acts, full64):
    """Every feasible logit is exactly 0: each step takes the lowest feasible index with log-prob -ln(#feasible)."""
    T = full64.shape[1] + 1
    feas = torch.isfinite(full64)                               # [R, T - 1, N]
    n = feas.sum(2)
    uniform = (-n.double().log())[..., None].expand_as(full64)
    assert torch.equal(full64[feas], uniform[feas]), "precondition: the oracle's feasible logits are not all 0"
    want = feas.int().argmax(2)                                 # lowest feasible index
    bad = (acts[:, 1:T] != want).nonzero()
    assert bad.numel() == 0, f"row, step {bad[0].tolist()}: tie not resolved to the lowest feasible index"
    torch.testing.assert_close(lp_gpu[:, 1:T].cpu(), -n.double().log().float(), rtol=0, atol=ATOL_LP)


def _zero_logit_key(pol):
    with torch.no_grad():
        pol.decoder.project_node_embeddings.weight[2 * E:3 * E] = 0.0


@pytest.mark.parametrize("N", [20, 50, 128])
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_exact_ties_through_an_eas_layer_resolve_to_the_lowest_index(env_name, N):
    """Lf = 0 (cache block 2): multistart greedy through a random EAS-Lay layer."""
    from rl4co_b200 import native

    B, S = 4, 5
    env, pol, td, td_host = _setup(env_name, N, B, seed=70 + N)
    _zero_logit_key(pol)
    hidden, cached, cache, _ = _cache(pol, td)
    assert not cache[..., 2 * E:3 * E].any()
    layer = _random_layer(B, seed=N)
    out = _layer_rollout(env_name, td, cached, cache, S, layer, mode=native.SELECT_GREEDY)
    acts = out["actions"].cpu()
    with torch.no_grad():
        _, full64 = _recorded_steps(teacher_forced_logprobs_with_layer, O.float64_weights(pol.state_dict(), ()),
                                    env_name, _td_host_dict(td_host), hidden.double().cpu(), acts,
                                    {k: v.detach() for k, v in _leaves(layer).items()}, num_starts=S, forced_first=True)
    _check_ties(out["logprobs"], acts, full64)


@pytest.mark.parametrize("N", [20, 50, 128])
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_exact_ties_through_a_poly_layer_resolve_to_the_lowest_index(env_name, N):
    """The un-folded logit key L = 0 (the POLY path reads it from cache block 2): multistart greedy through random poly
    weights."""
    k, S, B = 3, 9, 4
    env, pol, td, inst = _poly_setup(env_name, N, B, k, seed=80 + N)
    _zero_logit_key(pol)
    with torch.inference_mode():
        out = pol(td, env, phase="test", decode_type="greedy", num_starts=S, return_sum_log_likelihood=False,
                  return_hidden=True)
    acts = out["actions"].cpu()
    _, full64 = _oracle_steps(_w64(pol), env_name, inst, out["hidden"].double().cpu(), acts, S)
    _check_ties(out["log_likelihood"], acts, full64)
