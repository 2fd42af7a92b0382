"""Tensor helpers of the rollout path, same names / argument meaning as rl4co/utils/ops.py.

Pure layout helpers (batchify / unbatchify / gather_by_index / start-node selection) are
views and index arithmetic in torch on whatever device the data lives; the arithmetic op
(`get_tour_length`-based rewards) goes through the CUDA library (rl4co_b200.native).
"""

from __future__ import annotations

import math

import torch

from .tensordict import TensorDict


def _batchify_single(x, repeats: int):
    """rl4co/utils/ops.py:10-13: start-major repeat, flat index = r * B + b."""
    s = x.shape
    return x.expand(repeats, *s).contiguous().view(s[0] * repeats, *s[1:])


def batchify(x, shape):
    """rl4co/utils/ops.py:16-29"""
    shape = [shape] if isinstance(shape, int) else shape
    for s in reversed(shape):
        x = _batchify_single(x, s) if s > 0 else x
    return x


def _unbatchify_single(x, repeats: int):
    """rl4co/utils/ops.py:32-35"""
    s = x.shape
    return x.view(repeats, s[0] // repeats, *s[1:]).permute(1, 0, *range(2, len(s) + 1))


def unbatchify(x, shape):
    """rl4co/utils/ops.py:38-51: '(r b) ... -> b r ...'"""
    shape = [shape] if isinstance(shape, int) else shape
    for s in reversed(shape):
        x = _unbatchify_single(x, s) if s > 0 else x
    return x


def gather_by_index(src, idx, dim=1, squeeze=True):
    """rl4co/utils/ops.py:54-66"""
    expanded_shape = list(src.shape)
    expanded_shape[dim] = -1
    idx = idx.view(idx.shape + (1,) * (src.dim() - idx.dim())).expand(expanded_shape)
    squeeze = idx.size(dim) == 1 and squeeze
    return src.gather(dim, idx).squeeze(dim) if squeeze else src.gather(dim, idx)


def unbatchify_and_gather(x, idx, n: int):
    """rl4co/utils/ops.py:69-74"""
    x = unbatchify(x, n)
    return gather_by_index(x, idx, dim=idx.dim())


def get_num_starts(td, env_name=None) -> int:
    """rl4co/utils/ops.py:115-125 (tsp / cvrp / sdvrp / op rows)"""
    num_starts = td["action_mask"].shape[-1]
    if env_name in ("cvrp", "sdvrp", "op", "pctsp"):
        num_starts -= 1
    return num_starts


def select_start_nodes(td, env, num_starts: int):
    """rl4co/utils/ops.py:128-149 (tsp / depot-env rows)"""
    num_loc = env.generator.num_loc if hasattr(env.generator, "num_loc") else 0xFFFFFFFF
    sel = torch.arange(num_starts, device=td.device).repeat_interleave(td.shape[0]) % num_loc
    if env.name == "tsp":
        return sel
    sel = sel + 1
    if env.name == "op" and (td["action_mask"][..., 1:].float().sum(-1) < num_starts).any():
        # ops.py:150-160: some customers may be out of reach: resample the starts from the available ones
        sel = torch.multinomial(td["action_mask"][..., 1:].float(), num_starts, replacement=True) + 1
        sel = sel.t().reshape(-1)  # "b n -> (n b)"
    return sel


def get_tour_length_reward(locs, actions, with_depot: bool):
    """-get_tour_length(gather_by_index(locs, actions)) fused in one CUDA kernel
    (rl4co/utils/ops.py:54-90 as used by tsp/env.py:150-156 and cvrp/env.py:138-147)."""
    from . import native

    return native.tour_length(locs.contiguous(), actions.contiguous(), with_depot)


def dihedral_8_augmentation(xy):
    """rl4co/data/transforms.py:16-38 (aug-major: flat index = a * B + b)."""
    x, y = xy.split(1, dim=2)
    zs = ((x, y), (1 - x, y), (x, 1 - y), (1 - x, 1 - y), (y, x), (1 - y, x), (y, 1 - x), (1 - y, 1 - x))
    return torch.cat([torch.cat(z, dim=2) for z in zs], dim=0)


def symmetric_transform(x, y, phi, offset: float = 0.5):
    """rl4co/data/transforms.py:49-69: rotation by phi about (offset, offset), then x <-> y where phi > 2*pi."""
    x, y = x - offset, y - offset
    x_prime = torch.cos(phi) * x - torch.sin(phi) * y
    y_prime = torch.sin(phi) * x + torch.cos(phi) * y
    mask = phi > 2 * math.pi
    xy = torch.cat((x_prime, y_prime), dim=-1)
    xy = torch.where(mask, xy.flip(-1), xy)
    return xy + offset


def symmetric_angles(xy, num_augment: int, first_augment: bool = False):
    """rl4co/data/transforms.py:80-84: one angle in [0, 4*pi) per row of the batchified xy (torch's stream, same
    expression and call order), 0 for the first 1/num_augment rows unless first_augment."""
    phi = torch.rand(xy.shape[0], device=xy.device) * 4 * math.pi
    if not first_augment:
        phi[: xy.shape[0] // num_augment] = 0.0
    return phi


def symmetric_augmentation(xy, num_augment: int = 8, first_augment: bool = False):
    """rl4co/data/transforms.py:72-86 (aug-major: flat index = a * B + b)."""
    phi = symmetric_angles(xy, num_augment, first_augment)
    x, y = xy[..., [0]], xy[..., [1]]
    return symmetric_transform(x, y, phi[:, None, None])


def min_max_normalize(x):
    """rl4co/data/transforms.py:89-90: one min / max over the whole tensor."""
    return (x - x.min()) / (x.max() - x.min())


class StateAugmentation:
    """rl4co/data/transforms.py:105-151.

    `augment_fn` is "dihedral8" (num_augment must be 8), "symmetric" (a random rotation about (0.5, 0.5), reflected
    half of the time, any num_augment) or a callable fn(batchified feature, num_augment).  The default stays
    "dihedral8" (rl4co's is "symmetric"), so that existing callers keep the dihedral-8 augmentation POMO uses.
    On a CUDA fp32 [B, N, 2] feature both named laws run as one kernel from the un-batchified rows; elsewhere they
    run the reference's torch expressions.  The angles of "symmetric" are drawn from torch's generator as the
    reference draws them, so a seed gives the reference's tensors bit for bit on either device."""

    def __init__(self, num_augment: int = 8, augment_fn="dihedral8", first_aug_identity: bool = True,
                 normalize: bool = False, feats=None, **_):
        if not callable(augment_fn) and augment_fn not in ("dihedral8", "symmetric"):
            raise ValueError(f"Unknown augment_fn: {augment_fn}. Available options: 'symmetric', 'dihedral8' or a "
                             "custom callable")
        assert not (augment_fn == "dihedral8" and num_augment != 8), (
            "When using the `dihedral8` augmentation function, then num_augment must be 8")
        self.num_augment = num_augment
        self.augment_fn = augment_fn
        self.first_aug_identity = first_aug_identity
        self.normalize = normalize
        self.feats = ["locs"] if feats is None else feats

    def _augment(self, x, base):
        """Augmented [S*B, ...] feature from the batchified x; `base` is its un-batchified [B, ...] source, or None
        when x's rows are not S copies of it (a feature listed twice in feats)."""
        S = self.num_augment
        if callable(self.augment_fn):
            return self.augment_fn(x, S)
        if self.augment_fn == "dihedral8":
            first = x[: x.shape[0] // 8]  # transforms.py:40-46 augments the first 1/8 of the rows
            if first.is_cuda and first.dim() == 3 and first.shape[-1] == 2 and first.dtype == torch.float32:
                from . import native

                return native.dihedral8(first.contiguous())  # one kernel: 8 B read, 64 B written per node
            return dihedral_8_augmentation(first)
        if (base is not None and base.is_cuda and base.dim() == 3 and base.shape[-1] == 2
                and base.dtype == torch.float32):
            from . import native

            return native.symmetric_augment(base.contiguous(), symmetric_angles(x, S), S)  # per node: 8 B read, 8 S B written
        return symmetric_augmentation(x, S)

    def __call__(self, td: TensorDict) -> TensorDict:
        td_aug = batchify(td, self.num_augment)
        done = set()
        for feat in self.feats:
            if not self.first_aug_identity:
                # transforms.py:142,147 keep td_aug[feat][[B], 0], i.e. node 0 of row B (image 1 of instance 0), not
                # augmentation 0 as the reference's docstring says; reproduced as the reference computes it
                init_aug_feat = td_aug[feat][list(td.size()), 0].clone()
            aug_feat = self._augment(td_aug[feat], None if feat in done else td[feat])
            if self.normalize:
                aug_feat = min_max_normalize(aug_feat)
            if not self.first_aug_identity:
                aug_feat[list(td.size()), 0] = init_aug_feat
            td_aug.set(feat, aug_feat)
            done.add(feat)
        return td_aug
