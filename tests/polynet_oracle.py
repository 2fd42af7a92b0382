"""Float64 reference for PolyNet: the oracle's decode loop with rl4co's PolyNetAttention pointer
(rl4co/models/nn/attention.py, PolyNetAttention.forward).

`O.pointer_logits` is replaced by a version that applies g' = g + poly_layer_2(relu(poly_layer_1(cat(g, z)))) to the
glimpse g = project_out(heads) before the logit key.  The weights are read from the same dict as the rest of the
decoder (`decoder.pointer.poly_layer_{1,2}.*`, `decoder.pointer.binary_vectors`), so float64 leaves there give the
gradient by autograd.

Which bit vector a row takes:
  * `rollout_polynet` follows the reference literally: the glimpse is [B, S, E] in a multistart decode (the oracle
    unbatchifies the state like am/decoder.py:178-192) and row s of that axis takes binary_vectors[s % k]; a
    single-start decode has S = 1, so every row takes binary_vectors[0];
  * `teacher_forced_logprobs_polynet` replays the batchified rows j = s * B + b one query each, so the strategy is
    given per row: s % k by default, or an explicit [S * B] tensor."""

import math

import torch
import torch.nn.functional as F

from oracle import am_rollout_oracle as O


def poly_layer(weights, glimpse, z):
    """g + poly_layer_2(relu(poly_layer_1(cat(g, z))))"""
    x = torch.cat((glimpse, z.to(glimpse.dtype)), -1)
    u = F.relu(F.linear(x, O._w(weights, "pointer.poly_layer_1.weight"), O._w(weights, "pointer.poly_layer_1.bias")))
    return glimpse + F.linear(u, O._w(weights, "pointer.poly_layer_2.weight"), O._w(weights, "pointer.poly_layer_2.bias"))


def pointer_logits_polynet(row_strategy=None):
    """`O.pointer_logits` with the PolyNet layer.  `row_strategy` None: the reference's rule along glimpse axis 1;
    else [rows] int64, one strategy per row of a [rows, 1, E] glimpse."""

    def pointer_logits(weights, q, K, V, L, mask, num_heads=8):
        def heads(x):
            return x.view(*x.shape[:-1], num_heads, -1).transpose(-2, -3)

        attn_mask = mask.unsqueeze(1) if mask.ndim == 3 else mask.unsqueeze(1).unsqueeze(2)
        o = F.scaled_dot_product_attention(heads(q), heads(K), heads(V), attn_mask=attn_mask)
        o = o.transpose(-2, -3)
        o = o.reshape(*o.shape[:-2], -1)
        glimpse = F.linear(o, O._w(weights, "pointer.project_out.weight"))
        bv = O._w(weights, "pointer.binary_vectors")
        k, S = bv.shape[0], glimpse.shape[1]
        if row_strategy is None:  # attention.py: binary_vectors.repeat(ceil(S / k), 1)[:S], broadcast over the batch
            z = bv.repeat(math.ceil(S / k), 1)[:S][None].expand(glimpse.shape[0], S, bv.shape[1])
        else:
            assert S == 1 and row_strategy.shape == (glimpse.shape[0],)
            z = bv[row_strategy][:, None, :]
        glimpse = poly_layer(weights, glimpse, z)
        logits = torch.bmm(glimpse, L.squeeze(-2).transpose(-2, -1)).squeeze(-2) / math.sqrt(glimpse.size(-1))
        assert not torch.isnan(logits).any(), "Logits contain NaNs"
        return logits

    return pointer_logits


def _with_pointer(fn, row_strategy, *args, **kw):
    original = O.pointer_logits
    O.pointer_logits = pointer_logits_polynet(row_strategy)
    try:
        return fn(*args, **kw)
    finally:
        O.pointer_logits = original


def rollout_polynet(weights, env_name, inst, h, **kw):
    """`O.rollout` through the PolyNet pointer (multistart decode types: trajectory s takes strategy s % k)."""
    return _with_pointer(O.rollout, None, weights, env_name, inst, h, **kw)


def teacher_forced_logprobs_polynet(weights, env_name, inst, h, acts, num_starts=1, strategy=None, **kw):
    """`O.teacher_forced_logprobs` through the PolyNet pointer; row j = s * B + b takes strategy[j] (default s % k)."""
    B = h.shape[0]
    if strategy is None:
        k = O._w(weights, "pointer.binary_vectors").shape[0]
        strategy = (torch.arange(B * max(num_starts, 1)) // B) % k
    return _with_pointer(O.teacher_forced_logprobs, strategy, weights, env_name, inst, h, acts, num_starts=num_starts,
                         **kw)
