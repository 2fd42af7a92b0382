"""GPU: wgmma 3xTF32 GEMM (co_gemm_tf32x3) against a float64 reference; accuracy must be
fp32-class (a plain TF32 GEMM would be ~1e-3 relative and fail)."""

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, w, bias, residual, scale, shift, relu):
    c = a.double() @ w.double().t()
    if bias is not None:
        c = c + bias.double()
    if residual is not None:
        c = c + residual.double()
    if relu:
        c = c.clamp_min(0)
    if scale is not None:
        c = c * scale.double() + shift.double()
    return c


@pytest.mark.parametrize("M,K,Nout", [(128, 128, 128), (1000, 128, 384), (777, 512, 128), (4096, 128, 640), (130, 128, 512),
                                      (76877, 128, 640), (70001, 128, 128), (80000, 128, 384)])  # last 3: W-stationary path
@pytest.mark.parametrize("epi", ["plain", "bias_relu", "residual_affine"])
def test_gemm_tf32x3_matches_fp64(M, K, Nout, epi):
    from rl4co_b200 import native

    dev = torch.device("cuda:0")
    torch.manual_seed(M + K + Nout)
    a = torch.randn(M, K, device=dev)
    w = torch.randn(Nout, K, device=dev) / K ** 0.5
    bias = residual = scale = shift = None
    relu = False
    if epi == "bias_relu":
        bias, relu = torch.randn(Nout, device=dev), True
    if epi == "residual_affine":
        bias = torch.randn(Nout, device=dev)
        residual = torch.randn(M, Nout, device=dev)
        scale, shift = torch.rand(Nout, device=dev) + 0.5, torch.randn(Nout, device=dev)
    hi, lo = native.split_tf32(w)
    assert torch.equal(hi + lo, w)
    assert ((hi.view(torch.int32) & 0x1FFF) == 0).all()
    out = native.gemm_tf32x3(a, hi, lo, bias=bias, residual=residual, scale=scale, shift=shift, relu=relu)
    torch.cuda.synchronize()
    ref = _ref(a, w, bias, residual, scale, shift, relu)
    err = (out.double() - ref).abs().max().item()
    fp32 = torch.nn.functional.linear(a, w)  # cuBLAS fp32 SIMT for scale
    err32 = (_ref(a, w, None, None, None, None, False) - fp32.double()).abs().max().item()
    mag = ref.abs().max().item()
    assert err <= max(8 * err32, 4e-6 * mag), f"err {err:.3e} vs fp32 {err32:.3e} (|C| {mag:.2f})"


def test_gemm_strided_views_and_column_block_output():
    """A as a row-strided view and C written into a column block of a wider buffer (how the
    encoder / cache use it)."""
    from rl4co_b200 import native

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    big = torch.randn(300, 384, device=dev)
    a = big[:, 128:256]
    w = torch.randn(256, 128, device=dev) * 0.1
    hi, lo = native.split_tf32(w)
    outbuf = torch.zeros(300, 640, device=dev)
    native.gemm_tf32x3(a, hi, lo, out=outbuf[:, 128:384])
    ref = a.double() @ w.double().t()
    torch.testing.assert_close(outbuf[:, 128:384].double(), ref, rtol=1e-5, atol=1e-5)
    assert (outbuf[:, :128] == 0).all() and (outbuf[:, 384:] == 0).all()


@pytest.mark.parametrize("M", [1, 127, 128, 129, 1000, 132 * 128 + 77, 148 * 128 + 77, 40000])
@pytest.mark.parametrize("affine", [True, False])
def test_ffn_fused_vs_float64(M, affine):
    """co_ffn_fused (FF1 -> ReLU -> FF2 + skip + folded BatchNorm, hidden activation in registers) against a
    float64 evaluation of SkipConnection(MLP) + eval BatchNorm (nn/graph/attnnet.py:33-53).  M = 40 000 makes the
    persistent CTAs loop over several tiles (weight ring / accumulator phase wrap-around)."""
    from rl4co_b200 import native

    torch.manual_seed(M)
    dev = "cuda:0"
    x = torch.randn(M, 128, device=dev) * 1.3
    w1 = torch.randn(512, 128, device=dev) / 128 ** 0.5
    b1 = torch.randn(512, device=dev) * 0.1
    w2 = torch.randn(128, 512, device=dev) / 512 ** 0.5
    b2 = torch.randn(128, device=dev) * 0.1
    scale = (1 + 0.2 * torch.randn(128, device=dev)) if affine else None
    shift = (0.1 * torch.randn(128, device=dev)) if affine else None
    w1s, w2s = native.split_tf32(w1), native.split_tf32(w2)
    out = native.ffn_fused(x, native.ffn_tile_weights(w1s[0], w1s[1], w2s[0], w2s[1]), b1, b2, scale, shift)
    xd = x.double()
    ref = xd + torch.relu(xd @ w1.double().t() + b1.double()) @ w2.double().t() + b2.double()
    if affine:
        ref = ref * scale.double() + shift.double()
    # 3xTF32 with K = 128 and K = 512 reductions: fp32-class (a strict-fp32 GEMM chain has the same error level)
    torch.testing.assert_close(out.double(), ref, rtol=4e-5, atol=4e-5)


def test_encoder_fused_ffn_equals_split_path(monkeypatch):
    """The encoder with co_ffn_fused (default) and with the separate GEMMs (CO_FFN=split) agree to fp32 round-off."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(0)
    dev = "cuda:0"
    env = get_env("tsp", generator_params=dict(num_loc=100))
    pol = FusedAttentionModelPolicy(env_name="tsp", num_encoder_layers=3).to(dev).eval()
    td = env.reset(env.generator(300).to(dev))
    with torch.inference_mode():
        monkeypatch.setenv("CO_FFN", "split")
        h_split, _ = pol.encoder(td)
        monkeypatch.delenv("CO_FFN")
        h_fused, _ = pol.encoder(td)
    torch.testing.assert_close(h_fused, h_split, rtol=2e-5, atol=2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("B,N", [(7, 100), (3, 20), (5, 128), (2, 2), (700, 51)])
def test_instance_norm_matches_torch(B, N):
    """co_instance_norm == nn.InstanceNorm1d(E, affine=True) on x.permute(0, 2, 1) (rl4co/models/nn/ops.py:30-54)."""
    from rl4co_b200 import native

    dev = torch.device("cuda:0")
    torch.manual_seed(B * 31 + N)
    x = torch.randn(B, N, 128, device=dev) * 3.0 + 0.7
    m = torch.nn.InstanceNorm1d(128, affine=True).to(dev)
    with torch.no_grad():
        m.weight.uniform_(0.5, 1.5)
        m.bias.uniform_(-0.5, 0.5)
        ref = m(x.permute(0, 2, 1)).permute(0, 2, 1)
        ref64 = torch.nn.functional.instance_norm(x.double().permute(0, 2, 1), weight=m.weight.double(), bias=m.bias.double(),
                                                  eps=m.eps).permute(0, 2, 1)
        out = native.instance_norm(x, m.weight, m.bias, m.eps)
    torch.testing.assert_close(out.double(), ref64, rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=2e-6)
