"""GPU: the hot-path kernels on buffers of more than 2^31 floats, the size the headline batch (65 536 TSP-100 instances)
reaches: its 6 553 600 x 640 decoder cache and 6 553 600 x 384 encoder `Wqkv` output.  Past 2^31 floats an address
must be formed in 64 bits; a 32-bit product or byte offset corrupts only the instances behind that offset, which no
smaller test reaches.

Each case takes the smallest batch that puts its buffer past 2^31 floats.  The rows checked are derived from the
per-instance (per-row) float count P: for k = 29, 30, 31 the instance whose span holds float offset 2^k (the 2^31-,
2^32- and 2^33-byte boundaries), the last two instances and instance 0 as a control.  They are compared bitwise
against the same kernel on a contiguous copy of just those instances (the kernels' rows are batch-independent:
test_gpu_gemm_pipeline.py, test_gpu_rollout_sweep.py::test_persistent_loop_batch_composition), and against a float64
reference at the tolerances the suite uses for the same kernel.  Every test prints its peak device memory and wall
time.
"""

import time

import pytest
import torch

from oracle import am_rollout_oracle as O
from test_gpu_gemm_pipeline import _operands
from test_gpu_rollout_sweep import _check, _record_rollouts, _replay, _run

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
E = 128
GIB = 1 << 30


@pytest.fixture(autouse=True)
def _peak_memory_and_time(request):
    """Prints the test's peak device memory and wall time (shown with -rP)."""
    torch.zeros(1, device=DEV)  # the caching allocator keeps no statistics before its first allocation
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize(DEV)
    print(f"{request.node.name}: max_memory_allocated {torch.cuda.max_memory_allocated(DEV) / GIB:.2f} GiB, "
          f"wall {time.perf_counter() - t0:.1f} s")


def _require_free(need_bytes):
    """Skip unless `need_bytes` of device memory is free (other work may share the GPU)."""
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < need_bytes:
        pytest.skip(f"needs {need_bytes / GIB:.1f} GiB of free device memory, {free / GIB:.1f} GiB free")


def _boundary_instances(P, count):
    """Instance 0, the instances whose P-float span holds float offset 2^29, 2^30 and 2^31, and the last two."""
    assert count * P > 1 << 31, "the buffer does not reach past 2^31 floats"
    return sorted({0, *((1 << k) // P for k in (29, 30, 31)), count - 2, count - 1})


def _release():
    torch.cuda.synchronize(DEV)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------- 1. cache GEMM (K = 128)
@pytest.mark.parametrize("Nout,M", [(640, 3_360_000), (384, 5_600_000)])
def test_cache_gemm_past_2_31_output_floats(Nout, M):
    """C = A W^T + bias with M * Nout just past 2^31: the epilogue's row offsets into C (and the TMA rows of A) must
    be 64-bit.  Row windows are compared bitwise with the GEMM of just those rows, and with float64."""
    from rl4co_b200 import native

    _require_free(4 * M * (128 + Nout) + GIB // 2)
    a, w, hi, lo = _operands(M, Nout, seed=M + Nout)
    bias = torch.randn(Nout, device=DEV)
    out = native.gemm_tf32x3(a, hi, lo, bias=bias)
    windows = [(max(0, r - 64), min(M, r + 64)) for r in _boundary_instances(Nout, M)] + [(0, 128), (M - 300, M)]
    for r0, r1 in windows:
        part = native.gemm_tf32x3(a[r0:r1], hi, lo, bias=bias)
        assert torch.equal(part, out[r0:r1]), (r0, r1)
        ref = a[r0:r1].double() @ w.double().t() + bias.double()
        torch.testing.assert_close(out[r0:r1].double(), ref, rtol=1e-5, atol=1e-5, msg=f"rows {r0}..{r1}")
    del a, out, part
    _release()


# ------------------------------------------------------------------------------- 2. encoder attention
@pytest.mark.parametrize("variant,N,B", [("wgmma", 100, 56_000), ("simt", 64, 87_500)])
def test_encoder_mha_past_2_31_qkv_floats(variant, N, B, monkeypatch):
    """co_encoder_mha on a [B * N, 384] projection of more than 2^31 floats: each instance's qkv base offset must be
    64-bit.  Boundary instances against the kernel on just those instances (bitwise) and float64 SDPA."""
    from rl4co_b200 import native

    _require_free(4 * B * N * (384 + E) + GIB // 2)
    monkeypatch.setenv("CO_MHA_VARIANT", variant)
    g = torch.Generator(device=DEV).manual_seed(B * N)
    qkv = torch.randn(B * N, 384, device=DEV, generator=g).mul_(1.5)
    out = native.encoder_mha(qkv, B, N)
    idx = torch.tensor(_boundary_instances(N * 384, B), device=DEV)
    sub = qkv.view(B, N * 384)[idx].contiguous().view(-1, 384)
    del qkv
    got = out.view(B, N * E)[idx].view(-1, E)
    del out
    assert torch.equal(native.encoder_mha(sub, idx.numel(), N), got), "an instance's output depends on the batch"
    q, k, v = sub.view(-1, N, 3, 8, 16).permute(2, 0, 3, 1, 4).unbind(0)
    ref = torch.nn.functional.scaled_dot_product_attention(q.double(), k.double(), v.double()).transpose(1, 2)
    torch.testing.assert_close(got.double(), ref.reshape(-1, E), rtol=1e-5, atol=1e-5 if variant == "simt" else 2e-5)
    _release()


# ------------------------------------------------------------------------------- 3-4. persistent rollout kernels
ROLLOUT_CASES = [("tsp", 100, 33_600), ("cvrp", 101, 41_600)]  # cache widths 5E = 640 and 4E = 512


def _rollout_setup(env_name, N, B, seed):
    """Seeded policy, instances and encoder output h; the rollout cache from h.  Returns the device state, the CPU
    weights, the CPU instances and h's rows of the boundary instances (h itself is dropped)."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    W_cache = (5 if env_name == "tsp" else 4) * E
    _require_free(4 * B * N * (E + W_cache) + GIB // 2)
    torch.manual_seed(seed)
    env = get_env(env_name, generator_params=dict(num_loc=N if env_name == "tsp" else N - 1), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1).eval()
    W = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    pol = pol.to(DEV)
    td_host = env.generator(B)
    td = env.reset(td_host.to(DEV))
    h = torch.randn(B, N, E, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    with torch.inference_mode():
        cached = pol.decoder._precompute_cache(h)
    assert cached.rollout_cache.shape == (B, N, W_cache)
    idx = torch.tensor(_boundary_instances(N * W_cache, B))
    h_sub = h[idx.to(DEV)].cpu()
    del h
    inst = {k: v[idx] for k, v in td_host.items()}
    return td, cached, W, inst, h_sub, idx


def _greedy(env_name, td, cache, graph_ctx, cached, B, N, S):
    """native.rollout as test_gpu_eas.py::_rollout calls it, greedy, S forced starts when S > 1."""
    from rl4co_b200 import native

    vrp = env_name == "cvrp"
    return native.rollout(env_name, native.SELECT_GREEDY, cache, graph_ctx, cached.q_placeholder, cached.w_capacity,
                          td["locs"].contiguous(), td["demand"].contiguous() if vrp else None,
                          td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None, B, N, num_starts=S,
                          forced_start=S > 1, num_loc=N - (1 if vrp else 0), T_max=N if not vrp else 2 * (N - 1))


def _rollout_past_2_31(env_name, N, B, S):
    """Greedy over a cache of more than 2^31 floats; the boundary instances' trajectories (start-major rows
    s * B + b) against a rollout of just those instances (bitwise: actions, per-step log-probs, reward) and the
    prefix oracle."""
    td, cached, W, inst, h_sub, idx = _rollout_setup(env_name, N, B, seed=N + S)
    cache, gctx = cached.rollout_cache, cached.graph_context_or_none
    big = _greedy(env_name, td, cache, gctx, cached, B, N, S)
    n, d = idx.numel(), idx.to(DEV)
    sub_td = {k: td[k][d].contiguous() for k in ("locs", "demand", "vehicle_capacity") if k in td.keys()}
    small = _greedy(env_name, sub_td, cache[d].contiguous(), gctx[d].contiguous() if gctx is not None else None, cached,
                    n, N, S)
    del cache, cached, gctx
    rows = (torch.arange(S)[:, None] * B + idx[None]).reshape(-1).to(DEV)  # row s * n + j of `small`
    for key in ("actions", "logprobs", "reward", "log_likelihood"):
        assert torch.equal(big[key][rows], small[key]), f"{key} of the boundary instances depends on the batch"
    gpu = {"actions": big["actions"][rows].cpu(), "log_likelihood": big["logprobs"][rows].cpu(),
           "reward": big["reward"][rows].cpu()}
    del big, small, td
    _release()
    _check(gpu, _replay(W, env_name, inst, h_sub, gpu["actions"], num_starts=S, forced_first=S > 1), "greedy")


@pytest.mark.parametrize("env_name,N,B", ROLLOUT_CASES)
def test_rollout_kernel_past_2_31_cache_floats(env_name, N, B):
    """rollout_kernel (one trajectory per instance): every instance's cache row offset must be 64-bit."""
    _rollout_past_2_31(env_name, N, B, S=1)


@pytest.mark.parametrize("env_name,N,B", ROLLOUT_CASES)
def test_rollout_ms_kernel_past_2_31_cache_floats(env_name, N, B):
    """rollout_ms_kernel (S = 2 forced starts share an instance's cache)."""
    _rollout_past_2_31(env_name, N, B, S=2)


# ------------------------------------------------------------------------------- 5. stepping path
def test_stepping_path_past_2_31_cache_floats(monkeypatch):
    """N = 200 is past the fused node limit: co_pointer_logits / co_select_action through the policy read a
    16 800 x 200 x 640 cache.  Boundary instances against the prefix oracle."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    N, B = 200, 16_800
    _require_free(4 * B * N * (E + 5 * E) + GIB)
    torch.manual_seed(200)
    env = get_env("tsp", generator_params=dict(num_loc=N), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name="tsp", num_encoder_layers=1).eval()
    W = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    pol = pol.to(DEV)
    td_host = env.generator(B)
    h = torch.randn(B, N, E, device=DEV, generator=torch.Generator(device=DEV).manual_seed(200))
    launches = _record_rollouts(monkeypatch)
    out = _run(pol, env, td_host, h, decode_type="greedy")
    assert not launches, "N = 200 must take the stepping path"
    idx = torch.tensor(_boundary_instances(N * 5 * E, B))
    d = idx.to(DEV)
    gpu = {"actions": out["actions"][d].cpu(), "log_likelihood": out["log_likelihood"][d].cpu(),
           "reward": out["reward"][d].cpu()}
    h_sub = h[d].cpu()
    del out, h
    _release()
    inst = {k: v[idx] for k, v in td_host.items()}
    _check(gpu, _replay(W, "tsp", inst, h_sub, gpu["actions"]), "greedy")


# ------------------------------------------------------------------------------- 6. encoder inference chunks
def test_encoder_inference_chunks():
    """B = 2 * inference_chunk + 5: the eval-mode tensor-core encoder runs in three chunks; the rows on either side
    of each chunk edge and the last against O.encoder_forward and the encoder on just those instances."""
    from rl4co_b200.encoder import AttentionModelEncoder
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.tensordict import TensorDict

    C = AttentionModelEncoder.inference_chunk
    N, B = 10, 2 * C + 5
    _require_free(2 * GIB)
    torch.manual_seed(10)
    env = get_env("tsp", generator_params=dict(num_loc=N), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name="tsp").eval()
    W = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    pol = pol.to(DEV)
    assert pol.encoder.gemm == "tf32x3"
    td_host = env.generator(B)
    idx = torch.tensor([0, C - 1, C, 2 * C - 1, 2 * C, B - 1])
    sub_host = TensorDict({k: v[idx] for k, v in td_host.items()}, batch_size=[idx.numel()])
    with torch.inference_mode():
        h, _ = pol.encoder(env.reset(td_host.to(DEV)))
        got = h[idx.to(DEV)].cpu()
        del h
        h_sub, _ = pol.encoder(env.reset(sub_host.to(DEV)))
        inst = {k: v for k, v in sub_host.items()}
        h_ref, _ = O.encoder_forward(W, "tsp", O.env_reset("tsp", inst), num_layers=3)
    torch.testing.assert_close(got, h_ref, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(got, h_sub.cpu(), rtol=1e-6, atol=1e-6)
    _release()
