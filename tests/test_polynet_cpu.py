"""CPU: PolyNet -- the float64 oracle against the reference's recorded decodes (tests/golden/polynet_*.npz) and the live
reference, the bit-vector table, `state_dict` compatibility with rl4co's names, the rollout ABI / binding checks of the
`poly` fields, the Poppy mask and its tie rule, and the teacher-forced pass through the poly layer against the oracle
under autograd (CPU tensors: stock SDPA and Linear, what is checked is the glue)."""

import ctypes
import itertools
import math

import pytest
import torch

from conftest import name_seeded_weights
from oracle import am_rollout_oracle as O
from oracle import ref_standin
from polynet_oracle import rollout_polynet, teacher_forced_logprobs_polynet

E = 128


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
@pytest.mark.parametrize("S", [2, 7])
def test_oracle_vs_golden(golden, env_name, S):
    """Multistart greedy and teacher-forced replay of the reference's multistart sampling, k = 3 (strategies wrap at
    S = 7)."""
    g = golden(f"polynet_{env_name}20")
    W, inst, h = g.weights(), g.inst(), g["h"]
    out = rollout_polynet(W, env_name, inst, h, decode_type="multistart_greedy", num_starts=S)
    assert torch.equal(out["actions"], g[f"greedy{S}_actions"])
    torch.testing.assert_close(out["logprobs"], g[f"greedy{S}_logprobs"], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(out["reward"], g[f"greedy{S}_reward"], rtol=1e-6, atol=0)
    acts = g[f"sampling{S}_actions"]
    lp = teacher_forced_logprobs_polynet(W, env_name, inst, h, acts, num_starts=S, forced_first=True)
    ref = g[f"sampling{S}_logprobs"]
    torch.testing.assert_close(lp, ref[:, : lp.shape[1]], rtol=1e-5, atol=1e-6)


@pytest.mark.skipif(not ref_standin.reference_available(), reason="the reference tree is not present")
@pytest.mark.parametrize("env_name,k,S", [("tsp", 3, 5), ("cvrp", 5, 3), ("tsp", 1, 4)])
def test_oracle_vs_live_reference(env_name, k, S):
    ref = ref_standin.load()
    torch.manual_seed(11 + k)
    Env = ref.TSPEnv if env_name == "tsp" else ref.CVRPEnv
    env = Env(generator_params=dict(num_loc=15))
    pol = ref.AttentionModelPolicy(env_name=env_name, num_encoder_layers=1).eval()
    pol.decoder.pointer = ref.attention.PolyNetAttention(k, E, 256, 8, mask_inner=True, out_bias=False)
    with torch.no_grad():
        pol.decoder.pointer.poly_layer_2.weight.mul_(4.0)
    td0 = env.generator(batch_size=[3])
    with torch.inference_mode():
        td = env.reset(td0.clone())
        h, _ = pol.encoder(td)
        o = pol(td.clone(), env, phase="test", decode_type="multistart_greedy", num_starts=S,
                return_sum_log_likelihood=False)
        W = {k_: v.clone() for k_, v in pol.state_dict().items()}
        inst = {k_: td0[k_] for k_ in td0.keys()}
        got = rollout_polynet(W, env_name, inst, h, decode_type="multistart_greedy", num_starts=S)
    assert torch.equal(got["actions"], o["actions"])
    torch.testing.assert_close(got["logprobs"], o["log_likelihood"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("k", [1, 3, 128])
def test_binary_vectors_match_reference_table(k):
    from rl4co_b200.polynet import binary_vectors

    bits = math.ceil(math.log2(k))
    bv = binary_vectors(k)
    assert bv.shape == (k, bits)
    # row i is i in binary, most significant bit first
    want = torch.tensor([[(i >> (bits - 1 - b)) & 1 for b in range(bits)] for i in range(k)], dtype=torch.float32)
    assert torch.equal(bv, want.reshape(k, bits))
    if ref_standin.reference_available():
        att = ref_standin.load().attention.PolyNetAttention(k, E, 256, 8)
        assert torch.equal(bv, att.binary_vectors.detach())
    assert torch.equal(bv, torch.tensor(list(itertools.product([0, 1], repeat=bits))[:k], dtype=torch.float32)
                       .reshape(k, bits))


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_state_dict_names(golden, env_name):
    """A reference PolyNet decoder's state_dict loads strictly; an AM / POMO policy's loads with strict=False, missing
    exactly the poly keys."""
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.polynet import FusedPolyNetDecoder, FusedPolyNetPolicy

    g = golden(f"polynet_{env_name}20")
    ref_sd = {k[len("decoder."):]: v for k, v in g.weights().items()}
    dec = FusedPolyNetDecoder(k=3, env_name=env_name)
    assert set(dec.state_dict()) == set(ref_sd)
    dec.load_state_dict(ref_sd, strict=True)
    assert torch.equal(dec.pointer.poly_layer_1.weight, ref_sd["pointer.poly_layer_1.weight"])
    assert not dec.pointer.binary_vectors.requires_grad

    pol = FusedPolyNetPolicy(k=3, env_name=env_name, num_encoder_layers=1)
    pol2 = FusedPolyNetPolicy(k=3, env_name=env_name, num_encoder_layers=1)
    pol2.load_state_dict(pol.state_dict(), strict=True)
    am = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1, normalization="instance")
    res = pol.load_state_dict(am.state_dict(), strict=False)
    assert not res.unexpected_keys
    assert sorted(res.missing_keys) == sorted(
        "decoder.pointer." + n for n in ("binary_vectors", "poly_layer_1.weight", "poly_layer_1.bias",
                                         "poly_layer_2.weight", "poly_layer_2.bias"))


def test_policy_constructor():
    from rl4co_b200 import PolyNetPolicy
    from rl4co_b200.polynet import FusedPolyNetPolicy

    assert PolyNetPolicy is FusedPolyNetPolicy
    pol = FusedPolyNetPolicy(k=4, env_name="cvrp")
    assert (pol.train_decode_type, pol.val_decode_type, pol.test_decode_type) == ("sampling",) * 3
    assert pol.tanh_clipping == 10.0 and pol.decoder.pointer.poly_layer_1.in_features == E + 2
    with pytest.raises(NotImplementedError, match="MatNet"):
        FusedPolyNetPolicy(k=4, encoder_type="MatNet")
    with pytest.raises(NotImplementedError):
        FusedPolyNetPolicy(k=4, env_name="sdvrp")
    with pytest.raises(NotImplementedError):
        FusedPolyNetPolicy(k=4, poly_layer_dim=128)


def test_pack_layout():
    from rl4co_b200 import native
    from rl4co_b200.polynet import FusedPolyNetDecoder, pack_poly

    dec = FusedPolyNetDecoder(k=3, env_name="tsp")
    p = dec.pointer
    P = native.POLY_DIM
    packed = pack_poly(p)
    assert packed.shape == (native.POLY_FIXED_FLOATS + 3 * P,)
    o = 0
    for want in (p.project_out.weight.t(), p.poly_layer_1.weight[:, :E].t(), p.poly_layer_2.weight.t()):
        assert torch.equal(packed[o:o + want.numel()].view(want.shape), want)
        o += want.numel()
    assert torch.equal(packed[o:o + E], p.poly_layer_2.bias)
    c = packed[o + E:].view(3, P)
    for i in range(3):
        z = p.binary_vectors[i]
        want = p.poly_layer_1.bias + p.poly_layer_1.weight[:, E:] @ z
        torch.testing.assert_close(c[i], want.detach(), rtol=0, atol=1e-6)
    # block 2 of the cache is the un-folded logit key
    wl = dec.project_node_embeddings.weight[2 * E:]
    assert torch.equal(dec.fused_weight()[2 * E:3 * E], wl)


def _rollout_args(**over):
    from rl4co_b200 import native

    a = native.RolloutArgs()
    a.env_kind, a.select_mode, a.B_inst, a.num_starts = native.ENV_TSP, native.SELECT_SAMPLE_PHILOX, 0, 4
    a.N, a.T_max, a.num_loc, a.flags = 20, 20, 20, native.ROLLOUT_FORCED_START
    a.tanh_clipping, a.temperature = 10.0, 1.0
    for name in ("cache", "locs", "actions_out", "logp_out", "reward_out", "loglik_out", "poly"):
        setattr(a, name, 4096)
    a.poly_k = 3
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_rollout_args_poly_fields_follow_eas_layer():
    from rl4co_b200 import native

    R = native.RolloutArgs
    assert R.poly.offset == R.eas_layer.offset + 8
    assert R.poly_k.offset == R.poly.offset + 8 and R.reserved1.offset == R.poly_k.offset + 4
    assert ctypes.sizeof(R) == R.reserved1.offset + 4
    assert native.POLY_FIXED_FLOATS == E * E + 2 * E * native.POLY_DIM + E


@pytest.mark.parametrize("over,code", [
    (dict(), 0), (dict(env_kind=1), 0), (dict(poly=None, poly_k=0), 0), (dict(poly=None, num_starts=1), 0),
    (dict(poly_k=128), 0),
    (dict(num_starts=1), -2), (dict(env_kind=2), -2), (dict(env_kind=3), -2), (dict(env_kind=4), -2),
    (dict(eas_layer=4096), -2),
    (dict(poly=4100), -1), (dict(poly=4104, env_kind=1), -1), (dict(poly_k=0), -1), (dict(poly_k=-2), -1),
])
def test_rollout_poly_abi_argument_checks(over, code):
    from rl4co_b200 import native

    a = _rollout_args(**over)
    assert native.lib().co_rollout(ctypes.byref(a), None) == code, native.lib().co_last_error_string()


def test_poly_binding_checks_arguments():
    from rl4co_b200 import native

    cache = torch.zeros(2, 20, 5 * E)
    locs = torch.zeros(2, 20, 2)
    poly = torch.zeros(native.POLY_FIXED_FLOATS + 3 * native.POLY_DIM)
    args = ("tsp", native.SELECT_SAMPLE_PHILOX, cache, None, torch.zeros(E), None, locs, None, None, 2, 20)
    kw = dict(num_starts=4, forced_start=True, num_loc=20)
    with pytest.raises(NotImplementedError, match="multistart"):
        native.rollout(*args, num_starts=1, poly=poly, poly_k=3)
    with pytest.raises(NotImplementedError, match="EAS-Lay"):
        native.rollout(*args, **kw, poly=poly, poly_k=3, layer=torch.zeros(2, native.EAS_LAYER_FLOATS))
    with pytest.raises(ValueError, match="poly_k"):
        native.rollout(*args, **kw, poly=poly)
    with pytest.raises(ValueError, match="poly"):
        native.rollout(*args, **kw, poly=poly, poly_k=4)
    with pytest.raises(native.NativeLibraryError, match="CUDA"):
        native.rollout(*args, **kw, poly=poly, poly_k=3)


def test_poppy_mask_and_ties():
    from rl4co_b200.polynet import poppy_mask

    gen = torch.Generator().manual_seed(0)
    r = torch.randn(64, 9, generator=gen)
    ref = (-r).argsort(1).argsort(1) < 1  # polynet/model.py calculate_loss, tie-free rewards
    assert torch.equal(poppy_mask(r), ref)
    tied = torch.tensor([[1.0, 3.0, 3.0, 0.0], [2.0, 2.0, 2.0, 2.0], [-1.0, -5.0, -1.0, -1.0]])
    m = poppy_mask(tied)
    assert torch.equal(m.sum(1), torch.ones(3, dtype=torch.int64))
    assert m.float().argmax(1).tolist() == [1, 0, 0]  # the lowest index among the tied best rows


def _setup(env_name, n, B, k, seed):
    from rl4co_b200.envs import get_env
    from rl4co_b200.polynet import FusedPolyNetPolicy
    from rl4co_b200.tensordict import TensorDict

    pol = FusedPolyNetPolicy(k=k, env_name=env_name, num_encoder_layers=1, normalization="batch")
    sd = name_seeded_weights(pol.state_dict(), seed)
    sd["decoder.pointer.binary_vectors"] = pol.decoder.pointer.binary_vectors.detach().clone()
    sd["decoder.pointer.poly_layer_2.weight"] *= 4.0
    pol.load_state_dict(sd)
    pol.eval()
    W64 = O.float64_weights(pol.state_dict(), {n_ for n_, p in pol.named_parameters() if p.requires_grad})
    pol.double()
    gen = torch.Generator().manual_seed(seed)
    inst = {k_: v.double() for k_, v in O.generate_instances(env_name, B, n, generator=gen).items()}
    env = get_env(env_name, generator_params=dict(num_loc=n))
    td = env.reset(TensorDict(dict(inst), batch_size=[B]))
    return pol, env, td, inst, W64, gen


@pytest.mark.parametrize("env_name,k,S", [("tsp", 3, 7), ("cvrp", 3, 2), ("cvrp", 4, 4), ("tsp", 1, 3)])
def test_teacher_forced_pass_through_poly_layer(env_name, k, S):
    """`evaluate_log_likelihood` with a PolyNet decoder (float64 product) equals the oracle per step and in gradient,
    row s on strategy s % k; an explicit per-row strategy replays single rows."""
    from rl4co_b200.reinforce import evaluate_log_likelihood

    B = 4
    pol, env, td, inst, W64, gen = _setup(env_name, 16, B, k, seed=5 + S)
    h64, _ = O.encoder_forward(W64, env_name, O.env_reset(env_name, inst), num_layers=1)
    with torch.no_grad():
        acts = rollout_polynet(W64, env_name, inst, h64, decode_type="multistart_sampling", num_starts=S,
                               generator=gen)["actions"]
    adv = torch.randn(acts.shape[0], generator=gen, dtype=torch.float64)
    lp64 = teacher_forced_logprobs_polynet(W64, env_name, inst, h64, acts, num_starts=S, forced_first=True)
    (adv * lp64.sum(1)).sum().backward()
    h, _ = pol.encoder(td)
    lp = evaluate_log_likelihood(pol, td, env, acts, hidden=h, return_sum=False, forced_first=True)
    (adv * lp.sum(1)).sum().backward()
    T = lp64.shape[1]
    torch.testing.assert_close(lp[:, :T], lp64.detach(), rtol=0, atol=1e-9)
    rel, zero = O.gradient_errors({n_: p.grad for n_, p in pol.named_parameters() if p.requires_grad}, W64)
    assert all(e < 1e-7 for e in rel.values()), rel
    assert all(v == 0 for v in zero.values()), zero
    if k > 1:
        assert pol.decoder.pointer.poly_layer_1.weight.grad.abs().sum() > 0
    # one row per instance on an explicit strategy: row s of the multistart rollout, replayed on its own
    s = torch.tensor([S - 1, 0, S // 2, 1])[:B] % S
    rows = acts.view(S, B, -1)[s, torch.arange(B)]
    with torch.no_grad():
        one = evaluate_log_likelihood(pol, td, env, rows, hidden=h, return_sum=False, forced_first=True,
                                      strategy=s % k)
        full = lp.view(S, B, -1)[s, torch.arange(B)]
    torch.testing.assert_close(one, full, rtol=0, atol=1e-10)
