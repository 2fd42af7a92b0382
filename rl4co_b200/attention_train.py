"""Differentiable attention for the training step on the hand-written forward / backward kernels
(`co_attn_fwd` / `co_attn_bwd`, csrc/attn_train.cu) -- SURVEY.md section 8f-2.

  encoder self-attention under autograd     rl4co/models/nn/attention.py:110-134  (F.scaled_dot_product_attention)
  glimpse of the teacher-forced pass        rl4co/models/nn/attention.py:300-314, models/zoo/am/decoder.py:156-193

`F.scaled_dot_product_attention` in fp32 is what the reference runs here.  The functions below are autograd.Function wrappers: forward saves the
per-row log-sum-exp, backward recomputes the probabilities (no N x N tensor in memory).  CUDA only -- there is no
fallback inside this module; callers decide (shape limits: 8 heads x 16, keys <= 128, queries <= 256 per call).
"""

from __future__ import annotations

import torch

from . import native

E, H = native.EMBED_DIM, native.NUM_HEADS
MAX_KEYS, MAX_QUERIES = 128, 256


def supported(q_len: int, kv_len: int, embed_dim: int, num_heads: int, device) -> bool:
    return (torch.device(device).type == "cuda" and embed_dim == E and num_heads == H and kv_len <= MAX_KEYS
            and q_len >= 1)


def pack_mask(mask: torch.Tensor) -> torch.Tensor:
    """bool [B, M, N] (True = attend) -> int32 [B, M, 4]: bit n % 32 of word n // 32 is key n (little-endian bytes)."""
    B, M, N = mask.shape
    if N < MAX_KEYS:
        mask = torch.nn.functional.pad(mask, (0, MAX_KEYS - N))
    w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device=mask.device)
    by = (mask.view(B, M, MAX_KEYS // 8, 8).to(torch.uint8) * w).sum(-1, dtype=torch.uint8)   # [B, M, 16] bytes
    return by.contiguous().view(torch.int32)                                                  # [B, M, 4]


def _like(o, dO):
    """dO with o's strides (the kernels read both through one set of strides). `.contiguous()` is not enough: a size-1
    batch dimension may carry any stride, e.g. the gradient slice of one 256-query chunk of a single instance."""
    return dO if dO.stride() == o.stride() else torch.empty_like(o).copy_(dO)


class _Attention(torch.autograd.Function):
    """o = softmax(q k^T / 4 [masked]) v per head; q [B, M, E], k / v [B, N, E] (last dim contiguous, any row / batch
    stride that is a multiple of 4 floats -- column views of the fused cache are fine), mask words or None."""

    @staticmethod
    def forward(ctx, q, k, v, mask_words):
        B, M, _ = q.shape
        o = torch.empty(B, M, E, device=q.device, dtype=torch.float32)
        lse = torch.empty(B, H, M, device=q.device, dtype=torch.float32)
        native.attn_fwd(q, k, v, mask_words, o, lse)
        ctx.save_for_backward(q, k, v, o, lse, mask_words if mask_words is not None else torch.empty(0))
        ctx.has_mask = mask_words is not None
        return o

    @staticmethod
    def backward(ctx, dO):
        q, k, v, o, lse, mw = ctx.saved_tensors
        dO = _like(o, dO)
        dq = torch.empty(q.shape, device=q.device, dtype=torch.float32)
        dk = torch.empty(k.shape, device=q.device, dtype=torch.float32)
        dv = torch.empty(v.shape, device=q.device, dtype=torch.float32)
        native.attn_bwd(q, k, v, mw if ctx.has_mask else None, o, lse, dO, dq, dk, dv)
        return dq, dk, dv, None


class _SelfAttentionPacked(torch.autograd.Function):
    """Encoder form: qkv [B, N, 3E] packed ("three h d") -> o [B, N, E]; the gradient is written straight into one
    packed [B, N, 3E] tensor (no slice-backward passes)."""

    @staticmethod
    def forward(ctx, qkv):
        B, N, _ = qkv.shape
        o = torch.empty(B, N, E, device=qkv.device, dtype=torch.float32)
        lse = torch.empty(B, H, N, device=qkv.device, dtype=torch.float32)
        native.attn_fwd(qkv[..., :E], qkv[..., E:2 * E], qkv[..., 2 * E:], None, o, lse)
        ctx.save_for_backward(qkv, o, lse)
        return o

    @staticmethod
    def backward(ctx, dO):
        qkv, o, lse = ctx.saved_tensors
        dO = _like(o, dO)
        dqkv = torch.empty_like(qkv)
        native.attn_bwd(qkv[..., :E], qkv[..., E:2 * E], qkv[..., 2 * E:], None, o, lse, dO,
                        dqkv[..., :E], dqkv[..., E:2 * E], dqkv[..., 2 * E:])
        return dqkv


def attention(q, k, v, mask=None, mask_words=None):
    """Multi-head attention of q [B, M, E] against k / v [B, N, E] with an optional bool mask [B, M, N] (True =
    attend); queries beyond 256 per instance are processed in chunks (the gradients of k / v add up in autograd)."""
    if mask is not None and mask_words is None:
        mask_words = pack_mask(mask)
    M = q.shape[1]
    if M <= MAX_QUERIES:
        return _Attention.apply(q, k, v, mask_words)
    outs = []
    for lo in range(0, M, MAX_QUERIES):
        mw = mask_words[:, lo:lo + MAX_QUERIES].contiguous() if mask_words is not None else None
        outs.append(_Attention.apply(q[:, lo:lo + MAX_QUERIES], k, v, mw))
    return torch.cat(outs, 1)


def self_attention_packed(qkv):
    """qkv [B, N, 3E] (contiguous) -> [B, N, E]; N <= 128."""
    return _SelfAttentionPacked.apply(qkv.contiguous())

