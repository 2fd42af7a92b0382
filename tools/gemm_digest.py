"""sha256 of co_gemm_tf32x3 outputs for seeded inputs, at the decoder-cache shape and the encoder shapes, with every
epilogue variant.  Two builds compute the same bits exactly when their digests are equal.

    python tools/gemm_digest.py [--lib PATH] [--json FILE]

`--lib` loads another build of libcorollout.so (e.g. the parent commit's) instead of the package's.
"""
import argparse
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from rl4co_b200 import native  # noqa: E402

# (name, M, K, Nout, epilogue): the decoder cache at tsp100's batch, the encoder's projections at its node count
CASES = [
    ("cache_tsp100", 65536 * 100, 128, 640, "none"),
    ("cache_tail", 4096 * 50 + 77, 128, 640, "none"),
    ("qkv", 409600, 128, 384, "bias"),
    ("out_proj_skip", 409600, 128, 128, "bias_residual"),
    ("ffn1_relu", 409600, 128, 512, "bias_relu"),
    ("ffn2_skip_bn", 409600, 512, 128, "bias_residual_affine"),
    ("skip_bn_k128", 409600 + 3, 128, 128, "bias_residual_affine"),
    ("inplace_residual", 100003, 128, 128, "inplace"),
    ("small", 129, 128, 384, "bias_relu"),
]


def run_case(M, K, Nout, epi, seed):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g)
    w = torch.randn(Nout, K, device=dev, generator=g) / K ** 0.5
    hi, lo = native.split_tf32(w)
    bias = torch.randn(Nout, device=dev, generator=g)
    res = torch.randn(M, Nout, device=dev, generator=g) if "residual" in epi or epi == "inplace" else None
    scale = torch.rand(Nout, device=dev, generator=g) + 0.5
    shift = torch.randn(Nout, device=dev, generator=g)
    if epi == "none":
        out = native.gemm_tf32x3(a, hi, lo)
    elif epi == "bias":
        out = native.gemm_tf32x3(a, hi, lo, bias=bias)
    elif epi == "bias_relu":
        out = native.gemm_tf32x3(a, hi, lo, bias=bias, relu=True)
    elif epi == "bias_residual":
        out = native.gemm_tf32x3(a, hi, lo, bias=bias, residual=res)
    elif epi == "bias_residual_affine":
        out = native.gemm_tf32x3(a, hi, lo, bias=bias, residual=res, scale=scale, shift=shift)
    elif epi == "inplace":
        out = native.gemm_tf32x3(a, hi, lo, out=res, residual=res)
    else:
        raise ValueError(epi)
    torch.cuda.synchronize()
    return hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--lib", default=None, help="libcorollout.so to load instead of the package's")
    p.add_argument("--json", default=None, help="also write the digests here")
    a = p.parse_args()
    if a.lib:
        native.LIB_PATH = os.path.abspath(a.lib)
    digests = {}
    for i, (name, M, K, Nout, epi) in enumerate(CASES):
        digests[name] = run_case(M, K, Nout, epi, seed=1000 + i)
        print(f"{name:18s} M={M:8d} K={K:3d} N={Nout:3d} {epi:22s} {digests[name]}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(digests, f, indent=1)


if __name__ == "__main__":
    main()
