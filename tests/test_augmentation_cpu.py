"""CPU: `StateAugmentation` with rl4co's parameters (`augment_fn`, `first_aug_identity`, `normalize`, `feats`) equals
the reference's `StateAugmentation` (data/transforms.py:105-151) bit for bit on CPU TensorDicts under the same seed,
rejects what the reference rejects, and reflects at exactly the angles the reference does."""

import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import ref_standin

needs_ref = pytest.mark.skipif(not ref_standin.reference_available(), reason="reference tree not staged")


def _td(layout, B=6, N=20, seed=0, extra_feat=False):
    from rl4co_b200.tensordict import TensorDict

    g = torch.Generator().manual_seed(seed)
    if layout == "tsp":
        d = {"locs": torch.rand(B, N, 2, generator=g)}
    else:  # cvrp: depot is node 0 of locs (cvrp/env.py:_reset)
        d = {"locs": torch.cat((torch.rand(B, 1, 2, generator=g), torch.rand(B, N, 2, generator=g)), 1),
             "demand": torch.randint(1, 10, (B, N), generator=g).float() / 40,
             "vehicle_capacity": torch.ones(B, 1)}
    if extra_feat:
        d["targets"] = torch.rand(B, 7, 2, generator=g)
    return TensorDict(d, batch_size=[B])


def _both(seed, td, **kw):
    """(ours, reference) StateAugmentation(**kw) applied to clones of td after the same torch.manual_seed."""
    from rl4co_b200 import ops

    ref = ref_standin.load()
    torch.manual_seed(seed)
    ours = ops.StateAugmentation(**kw)(td.clone())
    torch.manual_seed(seed)
    theirs = ref.transforms.StateAugmentation(**kw)(td.clone())
    return ours, theirs


def _assert_same(ours, theirs):
    assert set(ours.keys()) == set(theirs.keys())
    assert ours.batch_size == theirs.batch_size
    for k in theirs.keys():
        assert ours[k].dtype == theirs[k].dtype and torch.equal(ours[k], theirs[k]), k


@needs_ref
@pytest.mark.parametrize("layout", ["tsp", "cvrp"])
@pytest.mark.parametrize("num_augment", [2, 8, 16])
@pytest.mark.parametrize("first_aug_identity", [True, False])
@pytest.mark.parametrize("normalize", [False, True])
def test_symmetric_equals_reference(layout, num_augment, first_aug_identity, normalize):
    td = _td(layout, seed=num_augment)
    ours, theirs = _both(7 + num_augment, td, num_augment=num_augment, augment_fn="symmetric",
                         first_aug_identity=first_aug_identity, normalize=normalize)
    _assert_same(ours, theirs)
    B = td.batch_size[0]
    if not normalize and first_aug_identity:
        # the first B rows have phi = 0: (x - 0.5) + 0.5, not the input itself, but never more than an ulp away
        torch.testing.assert_close(ours["locs"][:B], td["locs"], rtol=0, atol=2 ** -24)
        assert not torch.allclose(ours["locs"][B:2 * B], td["locs"], atol=1e-3)


@needs_ref
@pytest.mark.parametrize("layout", ["tsp", "cvrp"])
@pytest.mark.parametrize("feats", [["locs"], ["locs", "targets"], ["targets", "locs", "targets"]])
def test_symmetric_several_features_equal_reference(layout, feats):
    """Each listed feature draws its own angles, in list order; a feature listed twice is augmented twice."""
    td = _td(layout, extra_feat=True)
    ours, theirs = _both(3, td, num_augment=8, augment_fn="symmetric", feats=feats)
    _assert_same(ours, theirs)
    if len(feats) == 2:  # different angles for the two features: images 1.. are not rotated alike
        torch.manual_seed(3)
        only_locs = ref_standin.load().transforms.StateAugmentation(num_augment=8, augment_fn="symmetric")(td.clone())
        assert torch.equal(ours["locs"], only_locs["locs"])
        torch.manual_seed(3)
        only_t = ref_standin.load().transforms.StateAugmentation(num_augment=8, augment_fn="symmetric",
                                                                 feats=["targets"])(td.clone())
        assert not torch.equal(ours["targets"], only_t["targets"])


@needs_ref
@pytest.mark.parametrize("first_aug_identity", [True, False])
@pytest.mark.parametrize("normalize", [False, True])
def test_dihedral8_keywords_equal_reference(first_aug_identity, normalize):
    td = _td("cvrp")
    ours, theirs = _both(0, td, num_augment=8, augment_fn="dihedral8", first_aug_identity=first_aug_identity,
                         normalize=normalize)
    _assert_same(ours, theirs)


@needs_ref
def test_callable_augment_fn_equals_reference():
    def jitter(xy, n):  # uses torch's generator, so the call order matters too
        return xy * 0.5 + torch.rand(xy.shape[0] // n, *xy.shape[1:]).repeat(n, 1, 1)

    td = _td("tsp", extra_feat=True)
    ours, theirs = _both(5, td, num_augment=4, augment_fn=jitter, feats=["locs", "targets"], first_aug_identity=False)
    _assert_same(ours, theirs)


@needs_ref
def test_first_aug_identity_false_keeps_one_node_as_the_reference_does():
    """transforms.py:142,147 save and restore td_aug[feat][[B], 0]: node 0 of row B only."""
    from rl4co_b200 import ops

    td = _td("tsp", B=5)
    torch.manual_seed(1)
    a = ops.StateAugmentation(num_augment=4, augment_fn="symmetric", first_aug_identity=False)(td.clone())["locs"]
    torch.manual_seed(1)
    b = ops.StateAugmentation(num_augment=4, augment_fn="symmetric")(td.clone())["locs"]
    diff = (a != b).any(-1)
    assert diff.sum() == 1 and diff[5, 0]
    assert torch.equal(a[5, 0], td["locs"][0, 0])


def test_unknown_law_and_dihedral8_count_are_rejected():
    from rl4co_b200 import ops

    with pytest.raises(ValueError, match="Unknown augment_fn"):
        ops.StateAugmentation(augment_fn="rotate90")
    with pytest.raises(AssertionError):
        ops.StateAugmentation(num_augment=4, augment_fn="dihedral8")
    with pytest.raises(AssertionError):
        ops.StateAugmentation(num_augment=4)  # the default law is dihedral-8
    ops.StateAugmentation(num_augment=4, augment_fn="symmetric")
    ops.StateAugmentation(num_augment=3, augment_fn=lambda x, n: x)


def _boundary_angles():
    two_pi = np.float32(2 * math.pi)
    four_pi = np.float32(4 * math.pi)
    return torch.tensor([two_pi, np.nextafter(two_pi, np.float32(0)), np.nextafter(two_pi, np.float32(7)), 0.0,
                         np.nextafter(four_pi, np.float32(0))], dtype=torch.float32)


@needs_ref
def test_reflection_boundary_matches_reference():
    """phi > 2*pi compares in fp32: fp32(2*pi) (which is above 2*pi) does not reflect, its upper neighbour does."""
    from rl4co_b200 import ops

    ref = ref_standin.load().transforms
    phi = _boundary_angles()
    assert (phi > 2 * math.pi).tolist() == [False, False, True, False, True]
    g = torch.Generator().manual_seed(2)
    xy = torch.rand(5, 30, 2, generator=g)
    x, y = xy[..., [0]], xy[..., [1]]
    ours = ops.symmetric_transform(x, y, phi[:, None, None])
    assert torch.equal(ours, ref.symmetric_transform(x, y, phi[:, None, None]))
    # rows 2 and 4 are the mirror images (x <-> y) of an unreflected rotation
    rot = torch.cat((torch.cos(phi)[:, None, None] * (x - 0.5) - torch.sin(phi)[:, None, None] * (y - 0.5),
                     torch.sin(phi)[:, None, None] * (x - 0.5) + torch.cos(phi)[:, None, None] * (y - 0.5)), -1) + 0.5
    for r, reflected in enumerate([False, False, True, False, True]):
        assert torch.equal(ours[r], rot[r].flip(-1) if reflected else rot[r])
    # and the reference's own entry point, with the angle draw included
    for first in (False, True):
        torch.manual_seed(4)
        a = ops.symmetric_augmentation(xy.repeat(3, 1, 1), 3, first)
        torch.manual_seed(4)
        assert torch.equal(a, ref.symmetric_augmentation(xy.repeat(3, 1, 1), 3, first))


def test_symmetric_augment_abi_rejects_bad_arguments_without_a_gpu():
    from rl4co_b200 import native

    L = ctypes.CDLL(native.build())
    L.co_symmetric_augment.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.co_last_error_string.restype = ctypes.c_char_p
    fake = 256  # never dereferenced: the arguments are rejected before any launch
    assert L.co_symmetric_augment(None, fake, fake, 4, 8, 20, None) == -1
    assert b"null pointer" in L.co_last_error_string()
    assert L.co_symmetric_augment(fake, fake, None, 4, 8, 20, None) == -1
    for B, S, N in ((-1, 8, 20), (4, 0, 20), (4, 8, 0)):
        assert L.co_symmetric_augment(fake, fake, fake, B, S, N, None) == -1
        assert b"bad shape" in L.co_last_error_string()
    assert L.co_symmetric_augment(fake + 4, fake, fake, 4, 8, 20, None) == -1  # float2 loads need 8-byte alignment
    assert b"aligned" in L.co_last_error_string()
    assert L.co_symmetric_augment(fake, fake, fake, 0, 8, 20, None) == 0  # empty batch: nothing to launch


def test_native_symmetric_augment_refuses_cpu_tensors():
    from rl4co_b200 import native

    with pytest.raises(native.NativeLibraryError):
        native.symmetric_augment(torch.rand(2, 5, 2), torch.zeros(4), 2)
    with pytest.raises(ValueError):
        native.symmetric_augment(torch.rand(2, 5, 2), torch.zeros(5), 2)
