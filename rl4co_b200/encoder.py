"""Attention-model graph encoder (SURVEY.md section 8f-1, "next" row): stock PyTorch modules
with the reference's module tree so that a reference ``state_dict`` loads unchanged.

  AttentionModelEncoder   rl4co/models/zoo/am/encoder.py:12-87
  TSP/VRPInitEmbedding    rl4co/models/nn/env_embeddings/init.py:55-68,115-136
  GraphAttentionNetwork   rl4co/models/nn/graph/attnnet.py:16-106
  MultiHeadAttention      rl4co/models/nn/attention.py:64-134
  Normalization           rl4co/models/nn/ops.py:30-54
  MLP                     rl4co/models/nn/mlp.py:8-60

It runs once per instance.  Inference (no autograd, eval mode, CUDA): every nn.Linear runs on the
hand-written wgmma 3xTF32 GEMM (`co_gemm_tf32x3`; bias / ReLU / skip connection / eval-mode
BatchNorm folded into its epilogue) and the attention core on `co_encoder_mha` (wgmma scores
and P.V for N > 64), the FFN block on `co_ffn_fused`, instance normalisation on `co_instance_norm`
-- `_net_fused` below.  Still stock torch ops there: the K = 2 / 3 init embedding and the
graph-context mean + Linear of the decoder.  Under autograd (training) the stock Linear / norm modules
run (cuBLAS), with the attention core on the hand-written forward / backward kernels
(`co_attn_fwd` / `co_attn_bwd`, attention_train.py); without a graph but in train mode (batch
statistics) the attention core runs on `co_encoder_mha`.
"""

from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


class TSPInitEmbedding(nn.Module):
    def __init__(self, embed_dim, linear_bias=True):
        super().__init__()
        self.init_embed = nn.Linear(2, embed_dim, linear_bias)

    def forward(self, td):
        return self.init_embed(td["locs"])


class VRPInitEmbedding(nn.Module):
    def __init__(self, embed_dim, linear_bias=True, node_dim: int = 3):
        super().__init__()
        self.init_embed = nn.Linear(node_dim, embed_dim, linear_bias)
        self.init_embed_depot = nn.Linear(2, embed_dim, linear_bias)

    def forward(self, td):
        depot, cities = td["locs"][:, :1, :], td["locs"][:, 1:, :]
        depot_embedding = self.init_embed_depot(depot)
        node_embeddings = self.init_embed(torch.cat((cities, self._node_feature(td)), -1))
        return torch.cat((depot_embedding, node_embeddings), -2)

    @staticmethod
    def _node_feature(td):
        return td["demand"][..., None]


class OPInitEmbedding(VRPInitEmbedding):
    """init.py:254-280: depot (x, y); customers (x, y, prize) -- the module tree of VRPInitEmbedding."""

    @staticmethod
    def _node_feature(td):
        return td["prize"][..., 1:, None]  # the depot's entry is excluded


def _train_attention_on(x, n_keys: int, num_heads: int) -> bool:
    import os

    return (x.is_cuda and x.dtype == torch.float32 and torch.is_grad_enabled() and x.shape[-1] == 128 and num_heads == 8
            and n_keys <= 128 and os.environ.get("CO_TRAIN_ATTN", "fused") != "sdpa")


class PCTSPInitEmbedding(VRPInitEmbedding):
    """init.py:221-251: depot (x, y); customers (x, y, expected prize, penalty)."""

    def __init__(self, embed_dim, linear_bias=True):
        super().__init__(embed_dim, linear_bias, node_dim=4)

    @staticmethod
    def _node_feature(td):
        return torch.stack((td["expected_prize"], td["penalty"][..., 1:]), -1)


class SkipConnection(nn.Module):
    def __init__(self, module):
        super().__init__()
        self.module = module

    def forward(self, x):
        return x + self.module(x)


class MultiHeadAttention(nn.Module):
    def __init__(self, embed_dim: int, num_heads: int, bias: bool = True):
        super().__init__()
        self.num_heads = num_heads
        self.Wqkv = nn.Linear(embed_dim, 3 * embed_dim, bias=bias)
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=bias)

    def forward(self, x):
        B, N, _ = x.shape
        qkv = self.Wqkv(x)
        if _train_attention_on(x, N, self.num_heads):
            # autograd path of the training step: hand-written forward / backward (co_attn_fwd / co_attn_bwd) on the
            # packed projection instead of torch's fp32 mem-efficient SDPA; CO_TRAIN_ATTN=sdpa forces the stock op
            from . import attention_train

            return self.out_proj(attention_train.self_attention_packed(qkv))
        if (x.is_cuda and not torch.is_grad_enabled() and x.dtype == torch.float32 and x.shape[-1] == 128
                and self.num_heads == 8 and N <= 128):
            # no graph, but train-mode normalisation keeps the stock module tree (phase 1 of a chunked training step):
            # the attention core still runs on the forward kernel (co_encoder_mha)
            from . import native

            return self.out_proj(native.encoder_mha(qkv.reshape(B * N, -1).contiguous(), B, N).view(B, N, -1))
        q, k, v = qkv.view(B, N, 3, self.num_heads, -1).permute(2, 0, 3, 1, 4).unbind(0)
        out = F.scaled_dot_product_attention(q, k, v)
        return self.out_proj(out.transpose(1, 2).reshape(B, N, -1))


class Normalization(nn.Module):
    def __init__(self, embed_dim, normalization="batch"):
        super().__init__()
        cls = {"batch": nn.BatchNorm1d, "instance": nn.InstanceNorm1d}[normalization]
        self.normalizer = cls(embed_dim, affine=True)

    def forward(self, x):
        if isinstance(self.normalizer, nn.BatchNorm1d):
            return self.normalizer(x.reshape(-1, x.size(-1))).view(*x.size())
        return self.normalizer(x.permute(0, 2, 1)).permute(0, 2, 1)


class MLP(nn.Module):
    def __init__(self, input_dim: int, output_dim: int, num_neurons: list[int]):
        super().__init__()
        dims_in = [input_dim] + num_neurons
        dims_out = num_neurons + [output_dim]
        self.lins = nn.ModuleList(nn.Linear(i, o) for i, o in zip(dims_in, dims_out))

    def forward(self, xs):
        for lin in self.lins[:-1]:
            xs = F.relu(lin(xs))
        return self.lins[-1](xs)


class MultiHeadAttentionLayer(nn.Sequential):
    def __init__(self, embed_dim, num_heads=8, feedforward_hidden=512, normalization="batch"):
        super().__init__(
            SkipConnection(MultiHeadAttention(embed_dim, num_heads)),
            Normalization(embed_dim, normalization),
            SkipConnection(MLP(embed_dim, embed_dim, [feedforward_hidden] if feedforward_hidden > 0 else [])),
            Normalization(embed_dim, normalization),
        )


class GraphAttentionNetwork(nn.Module):
    def __init__(self, num_heads, embed_dim, num_layers, normalization="batch", feedforward_hidden=512):
        super().__init__()
        self.layers = nn.Sequential(*(MultiHeadAttentionLayer(embed_dim, num_heads, feedforward_hidden, normalization)
                                      for _ in range(num_layers)))

    def forward(self, x, mask=None):
        assert mask is None, "Mask not yet supported!"
        return self.layers(x)


class AttentionModelEncoder(nn.Module):
    def __init__(self, embed_dim: int = 128, init_embedding=None, env_name: str = "tsp", num_heads: int = 8,
                 num_layers: int = 3, normalization: str = "batch", feedforward_hidden: int = 512, net=None, **_):
        super().__init__()
        env_name = getattr(env_name, "name", env_name)
        self.env_name = env_name
        if init_embedding is None:
            init_embedding = {"tsp": TSPInitEmbedding, "cvrp": VRPInitEmbedding, "sdvrp": VRPInitEmbedding,
                              "op": OPInitEmbedding, "pctsp": PCTSPInitEmbedding}[env_name](embed_dim)
        self.init_embedding = init_embedding
        self.net = GraphAttentionNetwork(num_heads, embed_dim, num_layers, normalization, feedforward_hidden) \
            if net is None else net

    #: instances per forward chunk when no autograd graph is needed (bounds the FFN-hidden
    #: activation to chunk * N * 512 floats; exact because eval-mode norms are per element)
    inference_chunk = 65536
    #: "tf32x3": Linear layers run on the hand-written wgmma 3xTF32 GEMM (fp32-class accuracy)
    #: with bias / ReLU / skip connection / eval-mode BatchNorm folded into its epilogue -- CUDA,
    #: no-grad, eval only; "cublas": stock nn.Linear (strict fp32), always used under autograd.
    gemm = "tf32x3"

    def forward(self, td, mask=None):
        init_h = self.init_embedding(td)
        B = init_h.shape[0]
        no_graph = not (torch.is_grad_enabled() or self.training)
        fused = no_graph and self.gemm == "tf32x3" and init_h.is_cuda and isinstance(self.net, GraphAttentionNetwork)
        run = self._net_fused if fused else (lambda x: self.net(x, mask))
        if not no_graph or B <= self.inference_chunk:
            return run(init_h), init_h
        out = torch.empty_like(init_h)
        for lo in range(0, B, self.inference_chunk):
            out[lo:lo + self.inference_chunk] = run(init_h[lo:lo + self.inference_chunk])
        return out, init_h

    # ------------------------------------------------------------------ tensor-core inference path
    def _split(self, w, k_slices: int = 1):
        """(hi, lo) tf32 split of a weight, cached until the parameter is modified.  With
        `k_slices` > 1 returns a list of per-K-slice contiguous (hi, lo) pairs (split-K)."""
        from . import native

        cache = self.__dict__.setdefault("_split_cache", {})
        key = (id(w), k_slices)
        ver = (w._version, w.data_ptr())
        hit = cache.get(key)
        if hit is None or hit[0] != ver:
            if k_slices == 1:
                val = native.split_tf32(w)
            else:
                ks = w.shape[1] // k_slices
                val = [native.split_tf32(w[:, i * ks:(i + 1) * ks].contiguous()) for i in range(k_slices)]
            hit = (ver, val)
            cache[key] = hit
        return hit[1]

    def _ffn_tiled(self, w1, w2):
        """Pre-tiled (TMA-ready) image of an FFN block's split weights, cached until either parameter is modified."""
        from . import native

        cache = self.__dict__.setdefault("_ffn_cache", {})
        key = (id(w1), id(w2))
        ver = (w1._version, w1.data_ptr(), w2._version, w2.data_ptr())
        hit = cache.get(key)
        if hit is None or hit[0] != ver:
            s1, s2 = self._split(w1), self._split(w2)
            hit = (ver, native.ffn_tile_weights(s1[0], s1[1], s2[0], s2[1]))
            cache[key] = hit
        return hit[1]

    def _linear_splitk(self, x, lin, residual, aff):
        """out = affine(x @ W^T + b + residual) for K = k*128 through the W-stationary K=128 pipeline:
        k passes, each accumulating onto the previous partial via the epilogue's residual operand."""
        from . import native

        K = lin.weight.shape[1]
        n = K // 128
        parts = self._split(lin.weight, n)
        acc = None
        for i, (hi, lo) in enumerate(parts):
            last = i == n - 1
            a = x[:, i * 128:(i + 1) * 128]
            res = residual if i == 0 else acc
            acc = native.gemm_tf32x3(a, hi, lo, out=acc if i > 0 else None, bias=lin.bias if i == 0 else None,
                                     residual=res, scale=aff[0] if (last and aff is not None) else None,
                                     shift=aff[1] if (last and aff is not None) else None)
        return acc

    @staticmethod
    def _ffn_fusable(ffn):
        import os

        lins = ffn.lins
        return (os.environ.get("CO_FFN", "fused") != "split" and len(lins) == 2 and lins[0].bias is not None
                and lins[1].bias is not None and tuple(lins[0].weight.shape) == (512, 128)
                and tuple(lins[1].weight.shape) == (128, 512) and type(ffn) is MLP)  # MLP: ReLU between the two Linear

    @staticmethod
    def _apply_norm(norm, h, B, N, E):
        """Non-batch normalisation of the fused path: instance norm on co_instance_norm, anything else stock."""
        from . import native

        m = norm.normalizer
        if (isinstance(m, nn.InstanceNorm1d) and not m.track_running_stats and h.is_cuda and E == native.EMBED_DIM
                and h.dtype == torch.float32):
            return native.instance_norm(h.view(B, N, E), m.weight, m.bias, m.eps).view(B * N, E)
        return norm(h.view(B, N, E)).reshape(B * N, E).contiguous()

    @staticmethod
    def _bn_affine(norm):
        bn = norm.normalizer
        if not isinstance(bn, nn.BatchNorm1d):
            return None
        scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
        return scale.contiguous(), (bn.bias - bn.running_mean * scale).contiguous()

    def _net_fused(self, x):
        """GraphAttentionNetwork.forward (nn/graph/attnnet.py:97-106) with every nn.Linear on
        co_gemm_tf32x3; SkipConnection (nn/ops.py:9-15) = residual operand, eval BatchNorm
        (nn/ops.py:30-46) = per-channel scale/shift of the same epilogue."""
        from . import native

        B, N, E = x.shape
        h = x.reshape(B * N, E).contiguous()
        for layer in self.net.layers:
            mha, norm1, ffn, norm2 = layer[0].module, layer[1], layer[2].module, layer[3]
            qkv = native.gemm_tf32x3(h, *self._split(mha.Wqkv.weight), bias=mha.Wqkv.bias)
            if N <= 128 and mha.num_heads == native.NUM_HEADS and E == native.EMBED_DIM:
                att = native.encoder_mha(qkv, B, N)
            else:
                q, k, v = qkv.view(B, N, 3, mha.num_heads, -1).permute(2, 0, 3, 1, 4).unbind(0)
                att = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B * N, E)
            aff = self._bn_affine(norm1)
            if aff is not None:
                h = native.gemm_tf32x3(att, *self._split(mha.out_proj.weight), bias=mha.out_proj.bias, residual=h,
                                       scale=aff[0], shift=aff[1])
            else:
                h = native.gemm_tf32x3(att, *self._split(mha.out_proj.weight), bias=mha.out_proj.bias, residual=h)
                h = self._apply_norm(norm1, h, B, N, E)
            lins = ffn.lins
            aff = self._bn_affine(norm2)
            if self._ffn_fusable(ffn):
                # FF1 -> ReLU -> FF2 (+ skip, + folded BatchNorm) in one kernel: the [B*N, 512] hidden activation
                # stays in registers (co_ffn_fused); CO_FFN=split forces the separate GEMMs
                h = native.ffn_fused(h, self._ffn_tiled(lins[0].weight, lins[1].weight), lins[0].bias, lins[1].bias,
                                     scale=aff[0] if aff is not None else None, shift=aff[1] if aff is not None else None)
                if aff is None:
                    h = self._apply_norm(norm2, h, B, N, E)
                continue
            f = h
            for lin in lins[:-1]:
                f = native.gemm_tf32x3(f, *self._split(lin.weight), bias=lin.bias, relu=True)
            last = lins[-1]
            if last.weight.shape[1] % 128 == 0 and last.weight.shape[1] > 128:
                h = self._linear_splitk(f, last, h, aff)
            elif aff is not None:
                h = native.gemm_tf32x3(f, *self._split(last.weight), bias=last.bias, residual=h, scale=aff[0], shift=aff[1])
            else:
                h = native.gemm_tf32x3(f, *self._split(last.weight), bias=last.bias, residual=h)
            if aff is None:
                h = self._apply_norm(norm2, h, B, N, E)
        return h.view(B, N, E)
