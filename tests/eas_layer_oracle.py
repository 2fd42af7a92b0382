"""Float64 reference for the EAS-Lay layer gradient: the oracle's teacher-forced decode loop with rl4co's per-instance
residual layer on the head output (rl4co/models/zoo/eas/decoder.py:12-31, nn.py).

`teacher_forced_logprobs_with_layer` runs `O.teacher_forced_logprobs` with `O.pointer_logits` replaced by a version that
applies o' = o + (relu(o W1 + b1) W2 + b2) per row between the head concatenation and project_out; the layer tensors
are batchified like the encoder output for multistart rows.  Float64 leaves then give d(loss)/d(layer) by autograd
(rl4co/models/zoo/eas/search.py:163-169 makes exactly these tensors the parameters)."""

import math

import torch
import torch.nn.functional as F

from oracle import am_rollout_oracle as O


def pointer_logits_with_layer(layer):
    """`O.pointer_logits` with the EAS-Lay residual between the head concatenation and project_out.  `layer` holds
    W1 / W2 [B', E, E] ((in, out), as `torch.matmul(o, W1)`) and b1 / b2 [B', 1, E] for the B' rows of the decoder
    call."""

    def pointer_logits(weights, q, K, V, L, mask, num_heads=8):
        def heads(x):
            return x.view(*x.shape[:-1], num_heads, -1).transpose(-2, -3)

        attn_mask = mask.unsqueeze(1) if mask.ndim == 3 else mask.unsqueeze(1).unsqueeze(2)
        o = F.scaled_dot_product_attention(heads(q), heads(K), heads(V), attn_mask=attn_mask)
        o = o.transpose(-2, -3)
        o = o.reshape(*o.shape[:-2], -1)
        o = o + (torch.matmul(torch.relu(torch.matmul(o, layer["W1"]) + layer["b1"]), layer["W2"]) + layer["b2"])
        glimpse = F.linear(o, O._w(weights, "pointer.project_out.weight"))
        logits = torch.bmm(glimpse, L.squeeze(-2).transpose(-2, -1)).squeeze(-2) / math.sqrt(glimpse.size(-1))
        assert not torch.isnan(logits).any(), "Logits contain NaNs"
        return logits

    return pointer_logits


def teacher_forced_logprobs_with_layer(weights, env_name, inst, h, acts, layer, num_starts=1, **kw):
    """`O.teacher_forced_logprobs` through a per-instance EAS-Lay layer {"W1", "b1", "W2", "b2"} ([B, E, E] / [B, 1, E],
    batchified like the encoder output for multistart rows); float64 leaves give d(loss)/d(layer) by autograd."""
    rows = {k: (O.batchify(v, num_starts) if num_starts > 1 else v) for k, v in layer.items()}
    original = O.pointer_logits
    O.pointer_logits = pointer_logits_with_layer(rows)
    try:
        return O.teacher_forced_logprobs(weights, env_name, inst, h, acts, num_starts=num_starts, **kw)
    finally:
        O.pointer_logits = original
