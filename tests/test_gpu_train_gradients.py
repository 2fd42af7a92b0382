"""GPU: gradients of the training step against a float64 autograd oracle.

A training step samples with the forward-only rollout, recomputes the log-likelihood of the sampled actions with the
differentiable teacher-forced pass (`evaluate_log_likelihood`; encoder and glimpse attention on the hand-written
`co_attn_fwd` / `co_attn_bwd` kernels up to 128 keys) and backpropagates a REINFORCE loss. Every case here computes one
scalar loss twice on the GPU -- on the default path and with CO_TRAIN_ATTN=sdpa (stock SDPA + cuBLAS) -- and once on
the host with the oracle (`O.encoder_forward` + `O.teacher_forced_logprobs`) over float64 leaves of the same weights,
along the GPU's own trajectories, and compares per named parameter e = O.gradient_errors (relative Frobenius error):

  e_sdpa   <= E_SDPA                       glue / replay bugs, shared by both GPU paths
  e_kernel <= max(RATIO * e_sdpa, E_FLOOR) the kernels may be at most a small factor worse than torch's own fp32

and a parameter the float64 loss does not reach (gradient None or 0) must have none on the GPU either. Per-step log-probs
agree with the oracle's at the suite's 2e-5. Each case prints one GRADREPORT line with its worst values.

The loss is piecewise smooth: an FFN unit whose pre-activation lies within fp32 round-off of 0 may take either side of
its ReLU on the GPU, and one such unit moves the encoder gradients by ~1e-4 (pctsp at N = 64: float64 pre-activation
4.5e-8, fp32 forward error ~5e-7 on both paths, kernel path on the other side). The oracle therefore differentiates the
branch the GPU forward took: it is given each path's ReLU pattern (`_Branch`), and a unit may differ from the float64
forward's own sign only where the float64 pre-activation is below FLIP_BAND.

Parts: A single-start, all envs, action-mask width N in {20, 33, 64, 65, 128} (65 / 128 bracket the kernels' key-pair
split and their 128-key limit); B multistart and POMO (Q = S * T queries per instance in 256-query chunks); C whole
training steps (`reinforce_step`, with `micro_batch`, `pomo_step`); D the decoding parameters of
`policy(td, env, phase="train")` under autograd; E past the fused limits (N = 129; 2 * clip / T = 80), where the
stepping path must re-score its actions differentiably; F the attention kernels at their edges against float64.
"""

import math

import pytest
import torch

from conftest import name_seeded_weights
from oracle import am_rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ENVS = ["tsp", "cvrp", "sdvrp", "op", "pctsp"]
ATOL_LP = 2e-5
E_SDPA, RATIO, E_FLOOR = 1e-4, 4.0, 2e-5
FLIP_BAND = 1e-5  # |float64 pre-activation| of a ReLU unit the GPU may put on the other side of 0 (20x the fp32 error)


@pytest.fixture(autouse=True)
def _highest_matmul_precision():
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    yield
    torch.set_float32_matmul_precision(prev)


def _num_loc(env_name, N):
    """N is the action-mask width: it counts the depot of the depot envs."""
    return N - 1 if env_name in O.DEPOT_ENVS else N


def _setup(env_name, N, B, seed, **policy_kw):
    """Policy with name-seeded weights (non-trivial BatchNorm running statistics), instances, and the reset state."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2, **policy_kw)
    pol.load_state_dict(name_seeded_weights(pol.state_dict(), seed))
    pol = pol.to(DEV).eval()
    env = get_env(env_name, generator_params=dict(num_loc=_num_loc(env_name, N)), check_solution=False)
    torch.manual_seed(seed)
    td_host = env.generator(B)
    inst = {k: td_host[k] for k in td_host.keys()}
    return pol, env, env.reset(td_host.to(DEV)), inst


class _Branch:
    """The ReLU pattern of the GPU's differentiable encoder passes (one bool tensor per layer and pass, in call order),
    handed to the oracle's encoder passes in the same order; counts the units where it differs from the float64
    forward's own sign and keeps the largest float64 |pre-activation| among them."""

    def __init__(self, pol):
        self.masks, self.flips, self.band = [], 0, 0.0
        self._hooks = [layer[2].module.lins[0].register_forward_hook(self._record) for layer in pol.encoder.net.layers]

    def _record(self, module, inputs, out):
        if torch.is_grad_enabled():
            self.masks.append((out > 0).cpu())

    def remove(self):
        for h in self._hooks:
            h.remove()

    def take(self, n):
        assert len(self.masks) >= n, "the oracle runs more encoder passes than the GPU did"
        masks, self.masks = self.masks[:n], self.masks[n:]
        return masks

    def note(self, masks, pre):
        for m, x in zip(masks, pre):
            flip = m != (x > 0)
            self.flips += int(flip.sum())
            if flip.any():
                self.band = max(self.band, float(x[flip].abs().max()))


def _oracle(W64, env_name, inst, acts, coef, branch, num_starts=1, forced_first=False, norm="batch", batch_stats=False,
            **decode_kw):
    """float64 loss sum_i coef_i * ll_i of trajectories `acts` [B*S, T] (host tensors) on the GPU pass's ReLU branch,
    backpropagated into W64; returns the per-step log-probs."""
    masks, pre = branch.take(2), []
    h64, _ = O.encoder_forward(W64, env_name, O.env_reset(env_name, inst), num_layers=2, normalization=norm,
                               batch_stats=batch_stats, relu_masks=masks, pre_activations=pre)
    branch.note(masks, pre)
    lp64 = O.teacher_forced_logprobs(W64, env_name, inst, h64, acts, num_starts=num_starts, forced_first=forced_first,
                                     **decode_kw)
    (coef.double() * lp64.sum(1)).sum().backward()
    return lp64.detach()


def _compare(part, case, pol, run, oracle):
    """`run()` computes the loss on the GPU and calls backward (from its own copy of the reset state: the stepping path
    advances the state it is given); it returns (log-probs, data): per-step [B*S, T] or
    summed [B*S] log-probs (or None), and what the oracle needs. `oracle(W64, data, branch)` builds the same loss in
    float64 on the GPU pass's ReLU branch and returns its per-step log-probs. The oracle runs once per GPU path: the two paths may sample different trajectories."""
    from rl4co_b200 import native  # noqa: F401  (the library is loaded before the environment variable is flipped)

    sd = {k: v.detach().cpu().clone() for k, v in pol.state_dict().items()}
    names = [k for k, _ in pol.named_parameters()]
    errs, flips = {}, {}
    mp = pytest.MonkeyPatch()
    try:
        for path in ("sdpa", "kernel"):
            if path == "sdpa":
                mp.setenv("CO_TRAIN_ATTN", "sdpa")
            else:
                mp.delenv("CO_TRAIN_ATTN", raising=False)
            pol.zero_grad(set_to_none=True)
            branch = _Branch(pol)
            try:
                lp, data = run()
            finally:
                branch.remove()
            grads = {k: None if p.grad is None else p.grad.detach().clone() for k, p in pol.named_parameters()}
            W64 = O.float64_weights(sd, names)
            lp64 = oracle(W64, data, branch)
            assert not branch.masks, "the GPU ran encoder passes the oracle did not"
            assert branch.band <= FLIP_BAND, f"{path}: a ReLU unit at float64 pre-activation {branch.band:.1e} flipped"
            flips[path] = branch.flips
            lp = None if lp is None else lp.detach().double().cpu()
            if lp is None:
                pass
            elif lp.dim() == 1:  # a training step reports summed log-likelihoods: T steps of round-off
                torch.testing.assert_close(lp, lp64.sum(1), rtol=0, atol=ATOL_LP * 10)
            else:
                T = lp64.shape[1]
                torch.testing.assert_close(lp[:, :T], lp64, rtol=0, atol=ATOL_LP)
                assert (lp[:, T:] == 0).all(), "padding after the episode carries log-probability"
            rel, zero = O.gradient_errors(grads, W64)
            assert not any(zero.values()), f"{path}: gradient where the float64 loss has none: {zero}"
            errs[path] = rel
    finally:
        mp.undo()
    rk, rs = errs["kernel"], errs["sdpa"]
    bad_s = {k: e for k, e in rs.items() if not e <= E_SDPA}
    bad_k = {k: (e, rs[k]) for k, e in rk.items() if not e <= max(RATIO * rs[k], E_FLOOR)}
    wk, ws = max(rk.values()), max(rs.values())
    print(f"GRADREPORT part={part} case={case} e_kernel={wk:.3e} ({max(rk, key=rk.get)}) e_sdpa={ws:.3e} "
          f"({max(rs, key=rs.get)}) ratio={wk / ws:.2f} relu_flips={flips['kernel']}/{flips['sdpa']}")
    assert not bad_s, f"e_sdpa above {E_SDPA}: {bad_s}"
    assert not bad_k, f"e_kernel above max({RATIO} e_sdpa, {E_FLOOR}): {bad_k}"


def _advantages(rows, seed):
    return torch.randn(rows, generator=torch.Generator().manual_seed(seed))


def _teacher_forced_case(part, case, pol, env, td, inst, acts, S=1, forced_first=False, use_graph_context=True):
    """Fixed trajectories `acts` (device) and advantages: evaluate_log_likelihood vs the oracle's step loop."""
    from rl4co_b200.reinforce import evaluate_log_likelihood

    coef = _advantages(acts.shape[0], acts.shape[0] + acts.shape[1])
    acts_h = acts.cpu()

    def run():
        lp = evaluate_log_likelihood(pol, td, env, acts, return_sum=False)
        (coef.to(DEV) * lp.sum(1)).sum().backward()
        return lp, None

    def oracle(W64, _, branch):
        return _oracle(W64, env.name, inst, acts_h, coef, branch, num_starts=S, forced_first=forced_first,
                       use_graph_context=use_graph_context)

    _compare(part, case, pol, run, oracle)


# ------------------------------------------------------------------------------- A. single start
@pytest.mark.parametrize("env_name,N", [(e, n) for e in ENVS for n in (20, 33, 64, 65, 128)])
def test_single_start_gradients_vs_float64(env_name, N):
    B = 16
    pol, env, td, inst = _setup(env_name, N, B, seed=N)
    with torch.no_grad():
        acts = pol(td, env, phase="train", decode_type="sampling", seed=N)["actions"]
    _teacher_forced_case("A", f"{env_name}-{N}", pol, env, td, inst, acts)


# ------------------------------------------------------------------------------- B. multistart / POMO
@pytest.mark.parametrize("env_name,N,S,B,graph", [(e, 20, 4, 12, True) for e in ENVS]
                         + [("tsp", 50, 50, 4, False), ("cvrp", 51, 50, 4, False)])
def test_multistart_gradients_vs_float64(env_name, N, S, B, graph):
    """S forced starts: step 0 at log-prob 0, no placeholder query (W_placeholder gets no gradient). POMO (S = N
    starts, no graph context: project_fixed_context gets none): Q = S * T queries per instance run in 256-query chunks
    with a short last chunk, the K / V gradients adding up across chunks."""
    pol, env, td, inst = _setup(env_name, N, B, seed=S + N, use_graph_context=graph)
    with torch.no_grad():
        acts = pol(td, env, phase="train", decode_type="multistart_sampling", num_starts=S, seed=S)["actions"]
    assert acts.shape[0] == S * B
    _teacher_forced_case("B", f"{env_name}-{N}-S{S}", pol, env, td, inst, acts, S=S, forced_first=True,
                         use_graph_context=graph)


# ------------------------------------------------------------------------------- C. whole training steps
def _reinforce_case(part, case, pol, env, td, inst, micro_batch=None, norm="batch", seed=0):
    """reinforce_step in train mode with the mean baseline; max_grad_norm=0 and SGD(lr=0) leave the raw gradient in
    p.grad. The oracle's loss -(r - b) * ll / B over the step's own trajectories, reward and baseline; with
    `micro_batch` each chunk's encoder uses its own batch statistics."""
    from rl4co_b200.reinforce import get_reinforce_baseline, reinforce_step

    B = td.batch_size[0]

    def run():
        opt = torch.optim.SGD(pol.parameters(), lr=0.0)
        res = reinforce_step(pol, env, td.clone(), get_reinforce_baseline("mean"), opt, seed=seed, max_grad_norm=0,
                             micro_batch=micro_batch)
        bl = torch.as_tensor(res["bl_val"]).float().cpu()
        return res["log_likelihood"], (res["actions"].cpu(), res["reward"].cpu(), bl)

    def oracle(W64, data, branch):
        acts, reward, bl = data
        coef = -(reward - bl) / B
        spans = [(lo, min(lo + micro_batch, B)) for lo in range(0, B, micro_batch)] if micro_batch else [(0, B)]
        lps = [_oracle(W64, env.name, {k: v[lo:hi] for k, v in inst.items()}, acts[lo:hi], coef[lo:hi], branch, norm=norm,
                       batch_stats=norm == "batch") for lo, hi in spans]
        T = max(x.shape[1] for x in lps)
        return torch.cat([torch.nn.functional.pad(x, (0, T - x.shape[1])) for x in lps])

    _compare(part, case, pol, run, oracle)


@pytest.mark.parametrize("env_name", ENVS)
def test_reinforce_step_gradients_vs_float64(env_name):
    N = 20 if env_name == "tsp" else 21
    pol, env, td, inst = _setup(env_name, N, 32, seed=5)
    _reinforce_case("C", f"reinforce-{env_name}", pol, env, td, inst, seed=5)


@pytest.mark.parametrize("env_name,norm", [("tsp", "batch"), ("cvrp", "batch"), ("tsp", "instance"),
                                           ("cvrp", "instance")])
def test_reinforce_step_micro_batch_gradients_vs_float64(env_name, norm):
    """Chunks of 16 of a batch of 40 (a short last chunk): per-chunk BatchNorm statistics; with instance norm the
    chunked gradient is the unchunked one."""
    N = 20 if env_name == "tsp" else 21
    pol, env, td, inst = _setup(env_name, N, 40, seed=6, normalization=norm)
    _reinforce_case("C", f"micro-{env_name}-{norm}", pol, env, td, inst, micro_batch=16, norm=norm, seed=6)


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_pomo_step_gradients_vs_float64(env_name, monkeypatch):
    """pomo_step(phase="train"): S = all starts, shared baseline (the mean over an instance's starts), train-mode
    BatchNorm. The trajectories are read off the call to evaluate_log_likelihood."""
    from rl4co_b200 import reinforce

    N, B = 20, 8
    pol, env, td, inst = _setup(env_name, N, B, seed=8, use_graph_context=False)
    seen, real = [], reinforce.evaluate_log_likelihood

    def recorded(policy, td_, env_, actions, **kw):
        seen.append(actions.cpu())
        return real(policy, td_, env_, actions, **kw)

    monkeypatch.setattr(reinforce, "evaluate_log_likelihood", recorded)

    def run():
        torch.manual_seed(8)
        res = reinforce.pomo_step(pol, env, td, phase="train", optimizer=torch.optim.SGD(pol.parameters(), lr=0.0))
        r = res["reward"].cpu()                                          # [B, S]
        return None, (seen[-1], r)  # pomo_step reports no log-likelihoods

    def oracle(W64, data, branch):
        acts, r = data
        S = r.shape[1]
        coef = (-(r - r.mean(1, keepdim=True)) / (B * S)).t().reshape(-1)  # start-major rows s * B + b
        return _oracle(W64, env_name, inst, acts, coef, branch, num_starts=S, forced_first=True, batch_stats=True,
                       use_graph_context=False)

    _compare("C", f"pomo-{env_name}", pol, run, oracle)


# ------------------------------------------------------------------------------- D. decoding parameters under autograd
@pytest.mark.parametrize("clip,temp", [(10.0, 2.0), (3.0, 1.0), (25.0, 1.0)])
@pytest.mark.parametrize("S", [1, 4])
@pytest.mark.parametrize("env_name", ["tsp", "cvrp", "sdvrp"])
def test_policy_forward_under_autograd_vs_float64(env_name, S, clip, temp):
    """policy(td, env, phase="train") with grad on: the fused rollout samples, and its log_likelihood is re-scored by
    the teacher-forced pass with the call's temperature, tanh clipping and forced first step (S > 1)."""
    _policy_forward_case("D", env_name, 33, S, clip, temp)


def _policy_forward_case(part, env_name, N, S, clip, temp, B=12):
    pol, env, td, inst = _setup(env_name, N, B, seed=int(10 * clip + 100 * temp) + S)
    kw = dict(decode_type="multistart_sampling", num_starts=S) if S > 1 else dict(decode_type="sampling")
    coef = _advantages(B * S, S)

    def run():
        out = pol(td.clone(), env, phase="train", seed=3, temperature=temp, tanh_clipping=clip, return_sum_log_likelihood=False,
                  **kw)
        assert out["log_likelihood"].requires_grad
        (coef.to(DEV) * out["log_likelihood"].sum(1)).sum().backward()
        return out["log_likelihood"], out["actions"].cpu()

    def oracle(W64, acts, branch):
        return _oracle(W64, env_name, inst, acts, coef, branch, num_starts=S, forced_first=S > 1, temperature=temp,
                       tanh_clipping=clip)

    _compare(part, f"{env_name}-{N}-S{S}-clip{clip:g}-T{temp:g}", pol, run, oracle)


# ------------------------------------------------------------------------------- E. past the fused limits
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_reinforce_step_past_128_nodes_vs_float64(env_name):
    """N = 129: the encoder and the glimpse take SDPA under autograd, the sampling the stepping kernels."""
    pol, env, td, inst = _setup(env_name, 129, 8, seed=129)
    _reinforce_case("E", f"reinforce-{env_name}-129", pol, env, td, inst, seed=129)


@pytest.mark.parametrize("N,temp", [(129, 1.0), (50, 0.25)])
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_stepping_path_under_autograd_vs_float64(env_name, N, temp, monkeypatch):
    """N = 129, and 2 * clip / T = 80: policy(td, env, phase="train") decodes on the stepping kernels, and under autograd
    its log_likelihood must still carry the policy's gradient."""
    from rl4co_b200 import native

    launches = []
    real = native.rollout
    monkeypatch.setattr(native, "rollout", lambda *a, **k: launches.append(1) or real(*a, **k))
    n = N + (1 if env_name == "cvrp" and N == 50 else 0)
    for S in (1, 4):
        _policy_forward_case("E", env_name, n, S, 10.0, temp, B=8)
    assert not launches, "the whole-episode kernel ran"


@pytest.mark.parametrize("kw", [dict(top_k=3), dict(top_p=0.9), dict(return_entropy=True),
                                dict(decode_type="beam_search", beam_width=3)], ids=["top_k", "top_p", "entropy", "beam"])
def test_stepping_path_refuses_what_it_cannot_rescore_under_autograd(kw):
    """Under autograd the stepping path re-scores its actions with the teacher-forced pass; a decoding it cannot
    replay is an error there, and runs as before without a graph."""
    pol, env, td, _ = _setup("tsp", 20, 4, seed=1)
    kw = {"decode_type": "sampling", **kw}
    with pytest.raises(NotImplementedError, match="under autograd"):
        pol(td, env, phase="train", **kw)
    with torch.no_grad():
        out = pol(td, env, phase="train", **kw)
    assert torch.isfinite(out["log_likelihood"]).all()


# ------------------------------------------------------------------------------- F. attention kernels at their edges
def _attention64(q, k, v, mask=None):
    """float64 multi-head attention (8 heads x 16) with the kernels' defined behaviour for a fully masked row: output
    0, and no gradient through that row (stock SDPA returns NaN there)."""
    B, M, E = q.shape
    H = 8

    def heads(x):
        return x.reshape(B, x.shape[1], H, E // H).transpose(1, 2)

    s = heads(q) @ heads(k).transpose(-1, -2) / math.sqrt(E // H)
    if mask is None:
        p = torch.softmax(s, -1)
    else:
        live = mask.any(-1)[:, None, :, None]
        s = s.masked_fill(~mask[:, None], float("-inf")).masked_fill(~live, 0.0)
        p = torch.softmax(s, -1) * live
    return (p @ heads(v)).transpose(1, 2).reshape(B, M, E)


def _strided(B, R, scale, gen, pad=3):
    """[B, R, 128] view at column 128 of a taller, wider buffer: batch stride (R + pad) * 384, not R * row stride"""
    buf = (torch.randn(B, R + pad, 384, generator=gen) * scale).to(DEV)
    return buf[:, 1:R + 1, 128:256], buf


def _check_attention(q, k, v, mask, g, tol=2e-5):
    """o and the q / k / v gradients of the kernels against float64: e = ||x - x64|| / max(||x64||, 0.1 * scale), the
    scale being the size of the terms summed into x (||dO|| max|k| / 4 for dq, ||dO|| max|q| / 4 for dk), so that a
    gradient that cancels to ~0 (one allowed key: dq = 0) is held to the round-off of its terms."""
    from rl4co_b200 import attention_train as AT

    qs, ks, vs = (t.detach().clone().requires_grad_(True) for t in (q, k, v))
    o = AT.attention(qs, ks, vs, mask)
    (o * g).sum().backward()
    q64, k64, v64 = (t.detach().double().cpu().requires_grad_(True) for t in (q, k, v))
    o64 = _attention64(q64, k64, v64, None if mask is None else mask.cpu())
    g64 = g.double().cpu()
    (o64 * g64).sum().backward()
    scale = {"o": 0.0, "dq": g64.norm() * k64.abs().max() / 4, "dk": g64.norm() * q64.abs().max() / 4, "dv": 0.0}
    errs = {}
    for name, a, b in (("o", o, o64), ("dq", qs.grad, q64.grad), ("dk", ks.grad, k64.grad), ("dv", vs.grad, v64.grad)):
        a, b = a.detach().double().cpu(), b.detach()
        assert torch.isfinite(a).all(), name
        errs[name] = float((a - b).norm() / max(float(b.norm()), 0.1 * float(scale[name])))
        assert errs[name] <= tol, f"{name}: relative error {errs[name]:.2e}"
    return errs


@pytest.mark.parametrize("M", [1, 2, 3, 64, 65, 255, 256, 257, 513])
@pytest.mark.parametrize("N", [1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128])
def test_attention_sizes_vs_float64(N, M):
    """Every key-pair split and mask word (N), query-pair split and 256-query chunk (M), random masks with at least one
    key per row, zero upstream gradient on every fifth row after the first."""
    gen = torch.Generator().manual_seed(N * 1000 + M)
    B = 2
    q = (torch.randn(B, M, 128, generator=gen)).to(DEV)
    k, v = (torch.randn(B, N, 128, generator=gen).to(DEV) for _ in range(2))
    mask = torch.rand(B, M, N, generator=gen) < 0.6
    mask[torch.arange(B)[:, None], torch.arange(M)[None], torch.randint(0, N, (B, M), generator=gen)] = True
    g = torch.randn(B, M, 128, generator=gen)
    g[:, 1::5] = 0
    errs = _check_attention(q, k, v, mask.to(DEV), g.to(DEV))
    print(f"GRADREPORT part=F case=sizes-N{N}-M{M} " + " ".join(f"{n}={e:.2e}" for n, e in errs.items()))


@pytest.mark.parametrize("N", [1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128])
def test_self_attention_packed_sizes_vs_float64(N):
    """The encoder form (unmasked, M = N, packed [B, N, 3E] with a packed gradient)."""
    from rl4co_b200 import attention_train as AT

    gen = torch.Generator().manual_seed(N)
    qkv = torch.randn(3, N, 384, generator=gen).to(DEV).requires_grad_(True)
    g = torch.randn(3, N, 128, generator=gen).to(DEV)
    o = AT.self_attention_packed(qkv)
    (o * g).sum().backward()
    x64 = qkv.detach().double().cpu().requires_grad_(True)
    o64 = _attention64(x64[..., :128], x64[..., 128:256], x64[..., 256:])
    (o64 * g.double().cpu()).sum().backward()
    for a, b in ((o, o64), (qkv.grad, x64.grad)):
        assert float((a.detach().double().cpu() - b).norm() / b.norm()) <= 2e-5


BOUNDARY_KEYS = (0, 31, 32, 63, 64, 95, 96, 127)


@pytest.mark.parametrize("lowest", [False, True])
@pytest.mark.parametrize("N", [33, 65, 97, 128])
def test_attention_one_key_per_row_at_word_boundaries(N, lowest):
    """Row i may attend only key BOUNDARY_KEYS[i % 8] (those below N): o = v[key], dq = 0, dv[key] = sum of dO over its
    rows. `lowest`: the allowed key scores ~300 below every other key, so a mask bit read from the wrong word or lane
    (a row max over a masked key) underflows the row to 0."""
    gen = torch.Generator().manual_seed(N + lowest)
    keys = [j for j in BOUNDARY_KEYS if j < N]
    B, M = 2, 3 * len(keys) + 1
    q = torch.rand(B, M, 128, generator=gen) + 0.5        # positive: a negative key scores low for every query
    k = torch.randn(B, N, 128, generator=gen)
    if lowest:
        k[:, keys] = -20.0
    v = torch.randn(B, N, 128, generator=gen)
    mask = torch.zeros(B, M, N, dtype=torch.bool)
    for i in range(M):
        mask[:, i, keys[i % len(keys)]] = True
    g = torch.randn(B, M, 128, generator=gen)
    errs = _check_attention(q.to(DEV), k.to(DEV), v.to(DEV), mask.to(DEV), g.to(DEV))
    print(f"GRADREPORT part=F case=onekey-N{N}-lowest{int(lowest)} " + " ".join(f"{n}={e:.2e}" for n, e in errs.items()))


@pytest.mark.parametrize("scale", [7.0, 0.01], ids=["one-hot", "uniform"])
@pytest.mark.parametrize("N,M", [(128, 256), (65, 33), (20, 513)])
def test_attention_score_extremes_strided_views(N, M, scale):
    """|scores| ~ 50 (near one-hot rows) and ~1e-4 (near uniform), on q / k / v views whose batch stride is not rows
    x row stride (slices of taller buffers), B = 1 and B = 3."""
    for B in (1, 3):
        gen = torch.Generator().manual_seed(N + M + B)
        q, _ = _strided(B, M, scale, gen)
        k, _ = _strided(B, N, scale, gen)
        v, _ = _strided(B, N, 1.0, gen)
        assert q.stride(0) != M * q.stride(1)
        mask = (torch.rand(B, M, N, generator=gen) < 0.8)
        mask[..., N // 2] = True
        g = torch.randn(B, M, 128, generator=gen)
        errs = _check_attention(q, k, v, mask.to(DEV), g.to(DEV))
        print(f"GRADREPORT part=F case=extreme-N{N}-M{M}-s{scale:g}-B{B} " +
              " ".join(f"{n}={e:.2e}" for n, e in errs.items()))


@pytest.mark.parametrize("N,M", [(20, 40), (128, 300)])
def test_attention_fully_masked_row(N, M):
    """A row without an allowed key is the kernels' defined case (stock SDPA gives NaN): its output is 0, its q gradient
    a finite 0, and it changes nothing for the other rows or for dK / dV -- the same call without the dead rows gives the
    same outputs for the other rows and the same dK / dV."""
    from rl4co_b200 import attention_train as AT

    gen = torch.Generator().manual_seed(N + M)
    q, k, v = (torch.randn(2, R, 128, generator=gen).to(DEV) for R in (M, N, N))
    mask = torch.rand(2, M, N, generator=gen) < 0.5
    mask[..., 0] = True
    dead = [0, M // 2, M - 1]
    mask[:, dead] = False
    g = torch.randn(2, M, 128, generator=gen).to(DEV)
    _check_attention(q, k, v, mask.to(DEV), g)
    qs, ks, vs = (t.clone().requires_grad_(True) for t in (q, k, v))
    o = AT.attention(qs, ks, vs, mask.to(DEV))
    (o * g).sum().backward()
    assert (o[:, dead] == 0).all() and (qs.grad[:, dead] == 0).all()
    live = [i for i in range(M) if i not in dead]
    q2, k2, v2 = (t.clone().requires_grad_(True) for t in (q[:, live], k, v))
    o2 = AT.attention(q2, k2, v2, mask[:, live].to(DEV))
    (o2 * g[:, live]).sum().backward()
    torch.testing.assert_close(o[:, live], o2, rtol=0, atol=1e-6)
    torch.testing.assert_close(ks.grad, k2.grad, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(vs.grad, v2.grad, rtol=1e-5, atol=1e-6)
