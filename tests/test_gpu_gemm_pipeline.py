"""GPU: the K = 128 path of co_gemm_tf32x3 (TMA-fed A ring, register-A split, two accumulator sets whose epilogues
overlap the next tile's MMAs).  A row's result must not depend on which tile, CTA, ring stage or accumulator set
computed it, so row slices are compared bitwise against the whole product."""

import pytest
import torch

pytestmark = pytest.mark.gpu


def _groups(nout):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, sms // ((nout + 127) // 128))


def _operands(M, Nout, seed, K=128):
    from rl4co_b200 import native

    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g)
    w = torch.randn(Nout, K, device=dev, generator=g) / K ** 0.5
    hi, lo = native.split_tf32(w)
    return a, w, hi, lo


@pytest.mark.parametrize("Nout", [128, 384, 640])
def test_row_slices_are_bitwise_independent(Nout):
    from rl4co_b200 import native

    M = _groups(Nout) * 128 * 3 + 901
    a, _, hi, lo = _operands(M, Nout, seed=Nout)
    full = native.gemm_tf32x3(a, hi, lo)
    again = native.gemm_tf32x3(a, hi, lo)
    assert torch.equal(full, again)
    for r0, r1 in ((0, 1), (37, 200), (64, 64 + 129), (1000, 1000 + 128 * 7 + 5), (M - 300, M)):
        part = native.gemm_tf32x3(a[r0:r1], hi, lo)
        assert torch.equal(part, full[r0:r1]), (r0, r1)


@pytest.mark.parametrize("Nout", [128, 640])
@pytest.mark.parametrize("k,delta", [(1, -1), (1, 1), (2, 0), (3, -1), (4, 1)])
def test_ring_and_accumulator_wrap(Nout, k, delta):
    """M = g * 128 * k +- 1 for the launch's group count g: odd and even tile counts per CTA (the accumulator set of
    the last tile), ring phases that wrap, and a partial last tile."""
    from rl4co_b200 import native

    M = _groups(Nout) * 128 * k + delta
    a, w, hi, lo = _operands(M, Nout, seed=M)
    out = native.gemm_tf32x3(a, hi, lo)
    ref = a.double() @ w.double().t()
    torch.testing.assert_close(out.double(), ref, rtol=1e-5, atol=1e-5)
    tail = native.gemm_tf32x3(a[-5:], hi, lo)
    assert torch.equal(tail, out[-5:])


@pytest.mark.parametrize("M", [1, 5, 127])
def test_small_m(M):
    from rl4co_b200 import native

    a, w, hi, lo = _operands(M, 384, seed=7)
    out = native.gemm_tf32x3(a, hi, lo)
    assert out.shape == (M, 384)
    torch.testing.assert_close(out.double(), a.double() @ w.double().t(), rtol=1e-5, atol=1e-5)


def test_m_zero_is_a_no_op():
    """M = 0 returns before any tensor map is encoded (the map would reject a zero dimension) and writes nothing, for
    empty tensors (null data pointers) and for empty views of real buffers alike."""
    from rl4co_b200 import native

    _, _, hi, lo = _operands(4, 384, seed=5)
    dev = hi.device
    out = native.gemm_tf32x3(torch.empty(0, 128, device=dev), hi, lo)
    assert out.shape == (0, 384)
    buf = torch.full((3, 384), 7.0, device=dev)
    out = native.gemm_tf32x3(torch.randn(4, 128, device=dev)[4:], hi, lo, out=buf[3:], bias=torch.ones(384, device=dev))
    torch.cuda.synchronize()
    assert out.shape == (0, 384)
    assert (buf == 7).all()


def test_strided_a_and_column_block_output():
    """lda > K (A as a column slice of a wider buffer) and C written into a column block; the neighbours stay intact."""
    from rl4co_b200 import native

    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    M = _groups(256) * 128 + 333
    big = torch.randn(M, 512, device=dev)
    a = big[:, 256:384]
    w = torch.randn(256, 128, device=dev) / 128 ** 0.5
    hi, lo = native.split_tf32(w)
    outbuf = torch.full((M, 640), 7.0, device=dev)
    native.gemm_tf32x3(a, hi, lo, out=outbuf[:, 128:384])
    assert torch.equal(outbuf[:, 128:384], native.gemm_tf32x3(a.contiguous(), hi, lo))
    torch.testing.assert_close(outbuf[:, 128:384].double(), a.double() @ w.double().t(), rtol=1e-5, atol=1e-5)
    assert (outbuf[:, :128] == 7).all() and (outbuf[:, 384:] == 7).all()


def test_inplace_residual():
    """residual is out: every element reads its own old value before it is overwritten."""
    from rl4co_b200 import native

    M = _groups(128) * 128 * 2 + 17
    a, w, hi, lo = _operands(M, 128, seed=3)
    dev = a.device
    bias = torch.randn(128, device=dev)
    acc = torch.randn(M, 128, device=dev)
    expect = native.gemm_tf32x3(a, hi, lo, bias=bias, residual=acc.clone())
    native.gemm_tf32x3(a, hi, lo, out=acc, bias=bias, residual=acc)
    assert torch.equal(acc, expect)


@pytest.mark.parametrize("epi", ["bias_relu", "residual", "residual_affine"])
def test_epilogues_vs_float64(epi):
    from rl4co_b200 import native

    Nout = 384
    M = _groups(Nout) * 128 * 2 + 55
    a, w, hi, lo = _operands(M, Nout, seed=11)
    dev = a.device
    bias = torch.randn(Nout, device=dev)
    residual = torch.randn(M, Nout, device=dev) if epi != "bias_relu" else None
    scale, shift = (torch.rand(Nout, device=dev) + 0.5, torch.randn(Nout, device=dev)) if epi == "residual_affine" else (None, None)
    relu = epi == "bias_relu"
    out = native.gemm_tf32x3(a, hi, lo, bias=bias, residual=residual, scale=scale, shift=shift, relu=relu)
    ref = a.double() @ w.double().t() + bias.double()
    if residual is not None:
        ref = ref + residual.double()
    if relu:
        ref = ref.clamp_min(0)
    if scale is not None:
        ref = ref * scale.double() + shift.double()
    err = (out.double() - ref).abs().max().item()
    assert err <= 4e-6 * ref.abs().max().item() + 1e-6, err
