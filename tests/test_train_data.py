"""The shuffled order of the device training batches (tests/train_order_oracle.py), and DeviceRayBatches' refusals, without a
GPU."""
import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from tests import train_order_oracle as O

SIZES = [1, 2, 3, 5, 7, 31, 97, 1009, 8191, 8192, 8193, 65535, 65536, 65537, 100003]


@pytest.mark.parametrize("n", SIZES)
def test_order_is_a_bijection(n):
    for seed, epoch in ((0, 0), (7, 3), (2 ** 64 - 1, 2 ** 40)):
        o = O.order(n, seed, epoch)
        assert o.dtype == np.int64 and o.shape == (n,)
        assert np.array_equal(np.sort(o), np.arange(n))


def test_the_network_alone_is_a_bijection_of_the_power_of_two():
    for bits in range(0, 17):
        m = 1 << bits
        x = O.feistel(np.arange(m, dtype=np.uint64), m, O.round_keys(5, 1))
        assert np.array_equal(np.sort(x.astype(np.int64)), np.arange(m))


def test_order_depends_on_seed_and_epoch_and_shuffles():
    n = 100003
    a = O.order(n, 0, 0)
    assert np.array_equal(a, O.order(n, 0, 0))
    assert not np.array_equal(a, O.order(n, 0, 1))
    assert not np.array_equal(a, O.order(n, 1, 0))
    # a shuffle, not a near-identity: consecutive positions land far apart, and few pixels stay put
    assert np.count_nonzero(a == np.arange(n)) < 10
    assert np.median(np.abs(np.diff(a))) > n / 10


def test_permute_of_positions_matches_the_whole_order():
    n, seed, epoch = 65537, 11, 4
    full = O.order(n, seed, epoch)
    p = np.array([0, 1, 500, 65535, 65536])
    assert np.array_equal(O.permute(p, n, seed, epoch), full[p])


def _cams(n, w=8, h=6):
    K = [[10.0, 0.0, w / 2], [0.0, 10.0, h / 2], [0.0, 0.0, 1.0]]
    pose = [[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0]]
    return [hb.Camera(pose=pose, K=K, width=w, height=h) for _ in range(n)]


@pytest.mark.parametrize("option, value", [("use_patches", True), ("precrop_iters", 500), ("use_full_image", True),
                                           ("blur_radius", 2)])
def test_modes_other_than_the_default_are_refused(option, value):
    with pytest.raises(ValueError, match=option):
        hb.DeviceRayBatches(_cams(2), torch.zeros(2, 6, 8, 3, dtype=torch.uint8), 16, **{option: value})


def test_malformed_inputs_are_refused():
    img = torch.zeros(2, 6, 8, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="uint8"):
        hb.DeviceRayBatches(_cams(2), img.float(), 16)
    with pytest.raises(ValueError, match="uint8"):
        hb.DeviceRayBatches(_cams(2), [img[0].float(), img[1].float()], 16)
    with pytest.raises(ValueError, match="one size"):
        hb.DeviceRayBatches(_cams(2), [img[0], torch.zeros(5, 8, 3, dtype=torch.uint8)], 16)
    with pytest.raises(ValueError, match="camera grid's size"):
        hb.DeviceRayBatches(_cams(1) + _cams(1, w=9), img, 16)
    with pytest.raises(ValueError, match="cameras for"):
        hb.DeviceRayBatches(_cams(3), img, 16)
    with pytest.raises(ValueError, match=r"\[n, H, W, 3\]"):
        hb.DeviceRayBatches(_cams(2), torch.zeros(2, 6, 8, 4, dtype=torch.uint8), 16)
    with pytest.raises(ValueError, match="c_in"):
        hb.DeviceRayBatches(_cams(2), img, 16, c_in=7)
    with pytest.raises(ValueError, match="batch_size"):
        hb.DeviceRayBatches(_cams(2), img, 0)
